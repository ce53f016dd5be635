"""Cost of the depth filter of the enumerations, on bench.py's synthetic states.

For each state (n = 40 and 64, masks of mux depth 0..3, i.e. the full mask and 128 / 64 / 32
positions) and each width 3, 5, 7 it times with CUDA events, median of --reps runs after one
warm-up:
  count      the unfiltered count (max_matches = 0)
  loose      the filtered count at max_depth = SBG_DEPTH_BINS - 1, plus reading its histogram
  at_min     the filtered count at the minimum depth that histogram shows
  pick4096   a pick of 4,096 uniform ranks on the filtered cursor at the minimum depth
The gate depths come from a seeded random graph: gates 0..7 are inputs (depth 0), every later gate
takes two random earlier gates.  The 7-LUT counts run on the list the warm-up installs (phase 2
only).  Also printed: the totals and the minimum depth.

With --empty, also the empty-mask states of scripts/enum_time.py, where every candidate matches
(3-LUT and 7-LUT at n = 40, 5-LUT at n = 40 and 64).

    python scripts/enum_depth_time.py [--n 40 64] [--reps 3] [--empty]
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


def random_graph_depths(n, seed):
    """Depths of a seeded random graph of n gates: 8 inputs, then two-input gates."""
    rs = np.random.RandomState(seed)
    depth = np.zeros(n, dtype=np.uint16)
    for g in range(8, n):
        a, b = rs.choice(g, 2, replace=False)
        depth[g] = 1 + max(depth[a], depth[b])
    return depth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[40, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--empty", action="store_true",
                    help="also the empty-mask states of scripts/enum_time.py (n = 40, 64)")
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W, median of %d runs" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0), args.reps))
    print("%4s %5s %5s | %12s %9s | %9s %4s %12s %9s | %9s" % (
        "n", "mask", "width", "total", "count", "loose", "min", "at_min", "count", "pick4096"))
    for n in args.n:
        depth = random_graph_depths(n, 77 + n)
        for j, st in enumerate(bench.build_batch(n, 4, args.seed)):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            gate_order = np.random.RandomState(1000 * args.seed + j).permutation(n)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            table(eng, n, positions, depth, gate_order, st, (3, 5, 7), args)
    if args.empty:
        # the empty mask: every candidate matches (totals up to 4.6e11)
        for n, widths in ((40, (3, 5, 7)), (64, (5,))):
            st = bench.build_batch(n, 4, args.seed)[3]
            eng.load(bench._state(n, 1000 + n), st["target"], np.zeros(4, dtype=np.uint64), [])
            gate_order = np.random.RandomState(args.seed).permutation(n)
            table(eng, n, 0, random_graph_depths(n, 77 + n), gate_order, st, widths, args)
    eng.close()


def table(eng, n, positions, depth, gate_order, st, widths, args):
    """One line per width of the loaded state."""
    runs = {3: lambda k: eng.enumerate3(gate_order, k),
            5: lambda k: eng.enumerate5(st["order5"], k),
            7: lambda k: eng.enumerate7(st["outer"], st["middle"], k)}
    runs = {w: runs[w] for w in widths}
    for width, run in runs.items():
        eng.clear_depth_filter()
        ms_c, e = timed(lambda: run(0), args.reps)

        def loose():
            eng.set_depth_filter(depth, sb.SBG_DEPTH_BINS - 1)
            run(0)
            return eng.depth_counts()
        ms_l, hist = timed(loose, args.reps)
        assert int(hist.sum()) == e.total
        if e.total == 0:
            print("%4d %5d %5d | %12d %9.3f | %9.3f %4s %12s %9s | %9s" % (
                n, positions, width, 0, ms_c, ms_l, "-", "-", "-", "-"), flush=True)
            continue
        dmin = int(np.flatnonzero(hist)[0])

        def at_min():
            eng.set_depth_filter(depth, dmin)
            return run(0)
        ms_m, em = timed(at_min, args.reps)
        assert em.total == int(hist[dmin])
        ranks = np.random.default_rng(args.seed).choice(
            em.total, min(4096, em.total), replace=False)
        ms_p, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
        print("%4d %5d %5d | %12d %9.3f | %9.3f %4d %12d %9.3f | %9.3f" % (
            n, positions, width, e.total, ms_c, ms_l, dmin, em.total, ms_m, ms_p),
            flush=True)


if __name__ == "__main__":
    main()
