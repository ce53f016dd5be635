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

    python scripts/enum_time.py [--n 40 64] [--reps 3]
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
    args = ap.parse_args()
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    print("%s, %d SMs, power limit %s W" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0)))
    print("%4s %5s %4s | %8s %7s %7s %7s | %10s %9s %9s %9s | %11s %7s %9s %9s %9s" % (
        "n", "mask", "inb", "matches3", "scan3", "count3", "first3", "matches5", "search5",
        "count5", "first5", "matches7", "list", "search7", "count7", "first7"))
    for n in args.n:
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
    eng.close()


if __name__ == "__main__":
    main()
