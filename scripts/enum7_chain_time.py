"""Cost and yield of the 7-LUT chain enumeration (sbg_enum7_chain) next to the whole-space tree
enumeration (sbg_enum7_all), on bench.py's synthetic states.

For each state (n = 40 and 64: masks of mux depth 0..3, i.e. 256, 128, 64 and 32 positions) it
times with CUDA events, median of --reps runs after one warm-up:
  count_all    the tree's whole-space count (max_matches = 0), with its total
  count_chain  the chain's count (max_matches = 0), with its total and feasible count
  page_chain   a 4,096-match page at total / 2 on count_chain's cursor (sbg_enum_fetch)
  pick_chain   a pick of 4,096 uniform ranks on that cursor (sbg_enum_pick)
and, from both tuple-grouped enumerations (one record per gate set with a match), how many gate
sets have a tree match, a chain match, and a chain match but no tree match (chain_only): the
nodes where a three-LUT circuit exists that search_7lut cannot see.  The card's name and power
limit are printed first.

    python scripts/enum7_chain_time.py [--n 40 64] [--reps 3]
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

PAGE = 1 << 24


def gate_sets(eng, run, shift):
    """The ranks of the gate sets with a match: the tuple-grouped enumeration, paged out."""
    eng.set_grouping("tuple")
    try:
        e = run(0)
        out = [eng.fetch_matches(first, PAGE)["key"] >> np.uint64(shift)
               for first in range(0, e.total, PAGE)]
    finally:
        eng.set_grouping(None)
    return np.concatenate(out) if out else np.zeros(0, dtype=np.uint64)


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
    print("%4s %5s | %15s %10s | %10s %15s %11s | %10s %10s | %10s %10s %10s" % (
        "n", "mask", "total_all", "count_all", "feasible", "total_chain", "count_chain",
        "page_chain", "pick_chain", "tree_sets", "chain_sets", "chain_only"), flush=True)
    for n in args.n:
        for st in bench.build_batch(n, 4, args.seed):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            o, m = st["outer"], st["middle"]
            ms_ca, ea = timed(lambda: eng.enumerate7_all(o, m, 0), args.reps)
            ms_cc, ec = timed(lambda: eng.enumerate7_chain(o, m, 0), args.reps)
            total = ec.total
            ms_pg = ms_pk = float("nan")
            if total:
                ranks = np.random.default_rng(args.seed).integers(0, total, 4096)
                ms_pg, _ = timed(lambda: eng.fetch_matches(total // 2, 4096), args.reps)
                ms_pk, _ = timed(lambda: eng.pick_matches(ranks), args.reps)
            tree = gate_sets(eng, lambda k: eng.enumerate7_all(o, m, k), 23)
            chain = gate_sets(eng, lambda k: eng.enumerate7_chain(o, m, k), 24)
            only = np.setdiff1d(chain, tree).size
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            print("%4d %5d | %15d %10.3f | %10d %15d %11.3f | %10.3f %10.3f | %10d %10d %10d" % (
                n, positions, ea.total, ms_ca, ec.feasible, total, ms_cc, ms_pg, ms_pk,
                tree.size, chain.size, only), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
