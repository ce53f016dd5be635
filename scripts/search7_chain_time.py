"""Cost and effect of the first-chain search (sbg_search7_chain) and of the drop-in's opt-in chain
stage (SBG_LUT_CHAIN=1).  The card's name and power limit are printed first.

1. bench.py's states (n = 40 and 64; masks of 256, 128, 64 and 32 positions): sbg_search7, then
   sbg_search7_chain on the list sbg_search7 installed, both timed with CUDA events (median of --reps
   after one warm-up), with the list length and the chain's found / key.
2. The recorded search_7lut calls that found nothing (tests/golden/run_*.bin), with the orders their
   recorded RNG gives: how many have a chain, and the per-call time of sbg_search7_chain (the
   recorded state loaded and its list installed by sbg_search7 first, as the drop-in's node call
   does).
3. With oracle/_ref/sboxgates_gpu built: drop-in runs with and without SBG_LUT_CHAIN=1, one process
   per run, each under the committed seed: the LUT count of the last graph written, the wall time,
   the nodes that took a chain and the seconds spent in sbg_search7_chain (from SBG_SHIM_STATS).

    python scripts/search7_chain_time.py [--n 40 64] [--reps 5] [--timeout 600] [--no-dropin]
"""
import argparse
import glob
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _support as S  # noqa: E402
import bench  # noqa: E402
import sboxgates_b200 as sb  # noqa: E402
from enum_time import timed  # noqa: E402
from sboxgates_b200.rng import Xorshift1024  # noqa: E402

RUNS = [("des_s1.txt", ["-l", "-o", "0"], "seed1"), ("des_s1.txt", ["-l", "-o", "0"], "seed2"),
        ("crypto1_fa.txt", ["-l"], "seed1"), ("crypto1_fa.txt", ["-l"], "seed2"),
        ("crypto1_fb.txt", ["-l"], "seed1"), ("crypto1_fb.txt", ["-l"], "seed2"),
        ("crypto1_fc.txt", ["-l"], "seed1"), ("crypto1_fc.txt", ["-l"], "seed2"),
        ("rijndael.txt", ["-l", "-o", "0"], "seed1"), ("sodark.txt", ["-l", "-o", "0"], "seed1")]


def bench_states(eng, ns, reps, seed):
    print("1. bench.py's states: sbg_search7 and sbg_search7_chain on its list (ms)")
    print("%4s %5s | %8s %10s | %11s %5s %18s" % ("n", "mask", "list", "search7", "chain", "found",
                                                 "key"), flush=True)
    for n in ns:
        for st in bench.build_batch(n, 4, seed):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            o, m = st["outer"], st["middle"]
            ms7, r7 = timed(lambda: eng.search7(o, m), reps)
            msc, rc = timed(lambda: eng.search7_chain(o, m), reps)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            print("%4d %5d | %8d %10.3f | %11.3f %5d %18s" % (
                n, positions, rc.tuples_feasible, ms7, msc, rc.found,
                hex(rc.key) if rc.found else "-"), flush=True)


def recorded_calls(eng):
    calls = []
    for path in sorted(glob.glob(os.path.join(S.GOLDEN, "run_*.bin"))):
        for rec in S.read_records(path):
            if rec.which == 7 and not rec.found:
                calls.append(rec)
    found, ms = 0, []
    for rec in calls:
        outer, middle = sb.shuffled_orders7(Xorshift1024.from_state(rec.rng_s, rec.rng_p))
        eng.load(rec.tables, rec.target, rec.mask, rec.inbits_list())
        eng.search7(outer, middle)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = eng.search7_chain(outer, middle)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        found += int(res.found)
    print("2. recorded unmatched search_7lut calls: %d, with a chain: %d; sbg_search7_chain per call "
          "median %.3f ms, max %.3f ms" % (len(calls), found, float(np.median(ms)), max(ms)),
          flush=True)


def dropin(timeout):
    exe = os.path.join(S.REF_DIR, "sboxgates_gpu")
    if not os.path.exists(exe):
        print("3. drop-in: oracle/_ref/sboxgates_gpu not built")
        return
    print("3. drop-in runs (LUTs of the last graph written, wall s, chain nodes, chain s)")
    print("%-16s %-10s %5s | %6s %8s | %6s %8s %6s %8s" % (
        "sbox", "args", "seed", "LUTs", "wall", "LUTs+", "wall+", "nodes+", "chain_s+"), flush=True)
    for sbox, cli, seed in RUNS:
        row = []
        for chain in (False, True):
            env = dict(os.environ, SBG_SEEDFILE=os.path.join(S.GOLDEN, seed + ".bin"),
                       SBG_SHIM_STATS="1")
            if chain:
                env["SBG_LUT_CHAIN"] = "1"
            with tempfile.TemporaryDirectory() as tmp:
                t0 = time.time()
                try:
                    res = subprocess.run([exe] + cli + [os.path.join(S.REF_DIR, "sboxes", sbox)],
                                         cwd=tmp, env=env, capture_output=True, text=True,
                                         timeout=timeout)
                except subprocess.TimeoutExpired:
                    row.append(("timeout", "%.0f" % (time.time() - t0), "-", "-"))
                    continue
                wall = time.time() - t0
                files = sorted(glob.glob(os.path.join(tmp, "*.xml")))
                if res.returncode != 0 or not files:
                    row.append(("rc %d" % res.returncode, "%.2f" % wall, "-", "-"))
                    continue
                luts = os.path.basename(files[-1]).split("-")[1]
                m = re.search(r"7-LUT chain stage: \d+ calls ([0-9.]+) s, (\d+) nodes", res.stderr)
                row.append((str(int(luts)), "%.2f" % wall, m.group(2) if m else "-",
                            m.group(1) if m else "-"))
        (l0, w0, _, _), (l1, w1, c1, s1) = row
        print("%-16s %-10s %5s | %6s %8s | %6s %8s %6s %8s" % (
            sbox, " ".join(cli), seed, l0, w0, l1, w1, c1, s1), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[40, 64])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--timeout", type=float, default=600.0)
    ap.add_argument("--no-dropin", action="store_true")
    args = ap.parse_args()
    print("%s, %d SMs, power limit %s W" % (
        torch.cuda.get_device_name(0), torch.cuda.get_device_properties(0).multi_processor_count,
        bench.power_limit_w(0)), flush=True)
    eng = sb.LutEngine(0, stream=torch.cuda.current_stream().cuda_stream)
    bench_states(eng, args.n, args.reps, args.seed)
    recorded_calls(eng)
    eng.close()
    if not args.no_dropin:
        dropin(args.timeout)


if __name__ == "__main__":
    main()
