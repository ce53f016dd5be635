"""Cost of grouped enumeration (sbg_enum_set_grouping) next to the ungrouped count.

On the empty-mask states of scripts/enum_functions_time.py --empty (every candidate matches: the
5-LUT and 7-LUT at n = 40, the 5-LUT at n = 64) and, with --bench, on bench.py's n = 40 states
(masks of mux depth 0..3), it times with CUDA events, median of --reps runs after one warm-up:
  count     the ungrouped count (max_matches = 0)
  shape     the count under "shape" grouping (one per gate set and ordering row)
  tuple     the count under "tuple" grouping (one per gate set)
and, on the tuple cursor, a 4,096-group page at its middle rank and a pick of 4,096 uniform groups.
Totals are printed next to each time.  The 7-LUT counts run on the list the warm-up installs
(phase 2 only).

    python scripts/enum_groups_time.py [--reps 3] [--bench]
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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--bench", action="store_true", help="also bench.py's n = 40 masked states")
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W, median of %d runs; times in ms, totals in brackets" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0), args.reps))
    print("%4s %5s %5s | %-24s | %-24s | %-24s | %9s %9s" % (
        "n", "mask", "width", "count", "shape", "tuple", "page4096", "pick4096"))
    for n, widths in ((40, (5, 7)), (64, (5,))):
        st = bench.build_batch(n, 4, args.seed)[3]
        eng.load(bench._state(n, 1000 + n), st["target"], np.zeros(4, dtype=np.uint64), [])
        table(eng, n, 0, st, widths, args)
    if args.bench:
        for st in bench.build_batch(40, 4, args.seed):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            table(eng, 40, positions, st, (5, 7), args)
    eng.close()


def table(eng, n, positions, st, widths, args):
    """One line per width of the loaded state."""
    runs = {5: lambda k: eng.enumerate5(st["order5"], k),
            7: lambda k: eng.enumerate7(st["outer"], st["middle"], k)}
    for width in widths:
        run = runs[width]
        cells = []
        for grouping in (None, "shape", "tuple"):
            eng.set_grouping(grouping)   # stays set across the timed counts
            ms, e = timed(lambda: run(0), args.reps)
            cells.append("%10.3f [%12d]" % (ms, e.total))
        # the tuple cursor is the last one counted
        t = e.total
        page = pick = "-"
        if t:
            ms_f, _ = timed(lambda: eng.fetch_matches(t // 2, 4096), args.reps)
            ranks = np.random.default_rng(args.seed).choice(t, min(4096, t), replace=False)
            ms_p, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
            page, pick = "%9.3f" % ms_f, "%9.3f" % ms_p
        eng.set_grouping(None)
        print("%4d %5d %5d | %s | %9s %9s" % (n, positions, width, " | ".join(cells), page, pick),
              flush=True)


if __name__ == "__main__":
    main()
