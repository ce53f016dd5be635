"""Per-state kernel times of one bench step (n gates, the 8 states of step seed 1003): which of
the four families dominates at each mask depth, and how long the lists are.  With a
-DSBG_COUNT_FILTER build (SBG_LIB=...) every phase-1 launch also prints its F1 line: work units, and
the pair sieve's `sieve` (slowest lane's iterations, summed over chunks) next to `positions`, and
`exact` (chunks the sieve left to the cell loop) next to `chunks`."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import sboxgates_b200 as sb  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 40
eng = sb.LutEngine(0)
eng.set_timing(True)
for seed in (1003, 1004):
    states = bench.build_batch(n, 8, seed)
    for i, st in enumerate(states):
        eng.stage(i, st["tables"], st["target"], st["mask"], st["inbits"])
    for rep in range(2):
        for i, st in enumerate(states):
            r = eng.search_batch([dict(slot=i, order5=st["order5"], outer=st["outer"],
                                       middle=st["middle"])])[0]
            if rep == 1:
                print("seed %d state %d depth %d: ms5 %.3f filter %.3f order %.3f decomp %.3f | "
                      "5: found %d feasible %d | 7: found %d list %d swept %.3e"
                      % (seed, i, i % 4, eng.kernel_ms(0), eng.kernel_ms(1), eng.kernel_ms(2),
                         eng.kernel_ms(3), r.r5.found, r.r5.tuples_feasible, r.r7.found,
                         r.r7.tuples_feasible, r.r7.tuples_swept))
