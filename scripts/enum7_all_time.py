"""Cost of the whole-space 7-LUT enumeration (sbg_enum7_all) next to the list form and search7, on
bench.py's synthetic states.

For each state (n = 40 and 64: masks of mux depth 0..3, i.e. 256, 128, 64 and 32 positions) it
times with CUDA events, median of --reps runs after one warm-up:
  search7      the first-match search (phase 1 and phase 2)
  count7       the list form's count (max_matches = 0) on the list search7 left installed
  count_all    the whole-space count (max_matches = 0); with its total and feasible count
  tuple_all    the same under tuple grouping: the number of feasible gate sets with a match
  page_all     a 4,096-match page at total / 2 on count_all's cursor (sbg_enum_fetch)
  pick_all     a pick of 4,096 uniform ranks on that cursor (sbg_enum_pick)
Then the empty mask at n = 40 (every combination feasible, every position a match): the
tuple-grouped count, and with --empty-ungrouped the ungrouped count (4.6e11 matches at n = 40 x
70 rows x 65,536 positions per combination).  The card's name and power limit are printed first.

    python scripts/enum7_all_time.py [--n 40 64] [--reps 3] [--empty-ungrouped]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import sboxgates_b200 as sb  # noqa: E402
from enum_time import timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[40, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--empty-ungrouped", action="store_true",
                    help="also count the ungrouped empty-mask enumeration at n = 40")
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0)))
    print("%4s %5s | %7s %9s %9s | %10s %15s %10s | %10s %10s | %9s %9s" % (
        "n", "mask", "list", "search7", "count7", "feasible", "total_all", "count_all",
        "tuples", "tuple_all", "page_all", "pick_all"), flush=True)
    for n in args.n:
        for st in bench.build_batch(n, 4, args.seed):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            o, m = st["outer"], st["middle"]
            ms_s7, _ = timed(lambda: eng.search7(o, m), args.reps)
            ms_c7, e7 = timed(lambda: eng.enumerate7(o, m, 0), args.reps)
            eng.set_grouping("tuple")
            ms_tg, eg = timed(lambda: eng.enumerate7_all(o, m, 0), args.reps)
            eng.set_grouping(None)
            ms_ca, ea = timed(lambda: eng.enumerate7_all(o, m, 0), args.reps)
            total = ea.total
            ms_pg = ms_pk = float("nan")
            if total:
                ranks = np.random.default_rng(args.seed).integers(0, total, 4096)
                ms_pg, _ = timed(lambda: eng.fetch_matches(total // 2, 4096), args.reps)
                ms_pk, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            print("%4d %5d | %7d %9.3f %9.3f | %10d %15d %10.3f | %10d %10.3f | %9.3f %9.3f" % (
                n, positions, e7.feasible, ms_s7, ms_c7, ea.feasible, total, ms_ca, eg.total,
                ms_tg, ms_pg, ms_pk), flush=True)
    st = bench.build_batch(40, 4, args.seed)[0]
    eng.load(bench._state(40, 1040), st["target"], np.zeros(4, dtype=np.uint64), [])
    eng.set_grouping("tuple")
    ms, e = timed(lambda: eng.enumerate7_all(st["outer"], st["middle"], 0), 1)
    eng.set_grouping(None)
    print("n=40 empty mask, tuple grouping: %d gate sets (feasible %d), count %.1f ms"
          % (e.total, e.feasible, ms), flush=True)
    if args.empty_ungrouped:
        ms, e = timed(lambda: eng.enumerate7_all(st["outer"], st["middle"], 0), 1)
        print("n=40 empty mask, ungrouped: %d matches, count %.1f ms" % (e.total, ms), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
