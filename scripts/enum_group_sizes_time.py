"""Cost of group sizes (sbg_enum_group_sizes) next to the grouped pick of the same ranks.

On enum_groups_time.py's empty-mask states (every candidate matches: the 5-LUT and 7-LUT at n = 40,
the 5-LUT at n = 64) and bench.py's n = 40 32-position state, per width and grouping ("shape",
"tuple") it counts the grouped cursor, then times with CUDA events, median of --reps runs after one
warm-up:
  page   the sizes of a 4,096-group page at the cursor's middle rank, and the pick of those ranks
  uniform  the sizes of 4,096 uniform groups, and the pick of those ranks
Totals (groups) and the mean size of the uniform ranks are printed next to the times.  The 7-LUT
counts run on the list the warm-up installs (phase 2 only).

    python scripts/enum_group_sizes_time.py [--reps 3]
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
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W, median of %d runs; times in ms" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0), args.reps))
    print("%4s %5s %5s %6s | %9s | %10s %10s | %10s %10s | %12s" % (
        "n", "mask", "width", "group", "groups", "page size", "page pick", "unif size",
        "unif pick", "mean size"))
    for n, widths in ((40, (5, 7)), (64, (5,))):
        st = bench.build_batch(n, 4, args.seed)[3]
        eng.load(bench._state(n, 1000 + n), st["target"], np.zeros(4, dtype=np.uint64), [])
        table(eng, n, 0, st, widths, args)
    for st in bench.build_batch(40, 4, args.seed):
        positions = sum(bin(int(w)).count("1") for w in st["mask"])
        if positions == 32:
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            table(eng, 40, positions, st, (5, 7), args)
    eng.close()


def table(eng, n, positions, st, widths, args):
    """One line per width and grouping of the loaded state."""
    runs = {5: lambda k: eng.enumerate5(st["order5"], k),
            7: lambda k: eng.enumerate7(st["outer"], st["middle"], k)}
    for width in widths:
        for grouping in ("shape", "tuple"):
            eng.set_grouping(grouping)
            t = runs[width](0).total
            cells = []
            if t:
                page = np.arange(t // 2, min(t, t // 2 + 4096), dtype=np.uint64)
                unif = np.random.default_rng(args.seed).choice(t, min(4096, t), replace=False)
                for ranks in (page, unif):
                    ms_s, sizes = timed(lambda: eng.group_sizes(ranks), args.reps)
                    ms_p, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
                    cells += ["%10.3f %10.3f" % (ms_s, ms_p)]
                cells.append("%12.1f" % float(sizes.mean()))
            else:
                cells = ["%10s %10s" % ("-", "-")] * 2 + ["%12s" % "-"]
            print("%4d %5d %5d %6s | %9d | %s" % (n, positions, width, grouping, t,
                                                  " | ".join(cells)), flush=True)
        eng.set_grouping(None)


if __name__ == "__main__":
    main()
