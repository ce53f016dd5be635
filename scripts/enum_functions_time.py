"""Cost of the function filter of the enumerations, on bench.py's synthetic states.

For each state (n = 40 and 64, masks of mux depth 0..3, i.e. the full mask and 128 / 64 / 32
positions) and each width 3, 5, 7 it times with CUDA events, median of --reps runs after one
warm-up, each a full count (max_matches = 0; the filter is installed before the timed runs):
  count      unfiltered
  neutral    under a filter of all 256 functions in every role, passed explicitly
  om_aff     outer and middle affine, inner all 256 (7-LUT: the popcount path)
  in_aff     inner affine, outer and middle all 256 (7-LUT: the count pass runs the emit loop)
  g194       every role gate_functions(194) (AND, OR, XOR)
and, on the first of in_aff / g194 / om_aff with a match, a 4,096-match page at its middle rank
and a 4,096-rank pick.  Totals are printed next to each time.  The 7-LUT counts run on the list the
warm-up installs (phase 2 only).

With --empty, also the empty-mask states of scripts/enum_time.py, where every candidate matches
(3-LUT and 7-LUT at n = 40, 5-LUT at n = 40 and 64).

    python scripts/enum_functions_time.py [--n 40 64] [--reps 3] [--empty]
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

ALL = list(range(256))
AFF = sorted(sb.AFFINE_FUNCTIONS)
G194 = sorted(sb.gate_functions(194))
FILTERS = [("neutral", (ALL, ALL, ALL)), ("om_aff", (AFF, AFF, None)),
           ("in_aff", (None, None, AFF)), ("g194", (G194, G194, G194))]


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
    ap.add_argument("--empty", action="store_true",
                    help="also the empty-mask states of scripts/enum_time.py (n = 40, 64)")
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W, median of %d runs; times in ms, totals in brackets" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0), args.reps))
    print("%4s %5s %5s | %s | %9s %9s" % (
        "n", "mask", "width", " | ".join("%-22s" % c for c in ["count"] + [f for f, _ in FILTERS]),
        "page4096", "pick4096"))
    for n in args.n:
        for j, st in enumerate(bench.build_batch(n, 4, args.seed)):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            gate_order = np.random.RandomState(1000 * args.seed + j).permutation(n)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            table(eng, n, positions, gate_order, st, (3, 5, 7), args)
    if args.empty:
        for n, widths in ((40, (3, 5, 7)), (64, (5,))):
            st = bench.build_batch(n, 4, args.seed)[3]
            eng.load(bench._state(n, 1000 + n), st["target"], np.zeros(4, dtype=np.uint64), [])
            gate_order = np.random.RandomState(args.seed).permutation(n)
            table(eng, n, 0, gate_order, st, widths, args)
    eng.close()


def table(eng, n, positions, gate_order, st, widths, args):
    """One line per width of the loaded state."""
    runs = {3: lambda k: eng.enumerate3(gate_order, k),
            5: lambda k: eng.enumerate5(st["order5"], k),
            7: lambda k: eng.enumerate7(st["outer"], st["middle"], k)}
    for width in widths:
        run = runs[width]
        eng.clear_function_filter()
        ms, e = timed(lambda: run(0), args.reps)
        cells = ["%9.3f [%10d]" % (ms, e.total)]
        totals = {}
        for name, sets in FILTERS:
            eng.set_function_filter(*sets)   # stays installed across the timed counts
            ms, ef = timed(lambda: run(0), args.reps)
            cells.append("%9.3f [%10d]" % (ms, ef.total))
            totals[name] = ef.total
            if name == "neutral":
                assert ef.total == e.total
        page = pick = "-"
        for name in ("in_aff", "g194", "om_aff"):
            if totals[name] == 0:
                continue
            eng.set_function_filter(*dict(FILTERS)[name])
            t = run(0).total
            ms_f, _ = timed(lambda: eng.fetch_matches(t // 2, 4096), args.reps)
            ranks = np.random.default_rng(args.seed).choice(t, min(4096, t), replace=False)
            ms_p, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
            page, pick = "%9.3f" % ms_f, "%9.3f" % ms_p
            break
        eng.clear_function_filter()
        print("%4d %5d %5d | %s | %9s %9s" % (n, positions, width, " | ".join(cells), page, pick),
              flush=True)


if __name__ == "__main__":
    main()
