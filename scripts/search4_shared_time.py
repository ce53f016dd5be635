"""Cost and effect of the shared-input two-LUT search (sbg_search4_shared, sbg_enum4_shared) and of
the drop-in's opt-in stage (SBG_LUT_SHARED=1).  The card's name and power limit are printed first.

1. bench.py's states (n = 40 and 64; masks of 256, 128, 64 and 32 positions): sbg_search5, then
   sbg_search4_shared and the counting sbg_enum4_shared under the same order, timed with CUDA events
   (median of --reps after one warm-up), with the feasible 4-combinations, the total and the first
   key.
2. The recorded search_5lut calls that found nothing (tests/golden/run_*.bin), with the order their
   recorded RNG gives: how many have a shared-input circuit, and the per-call time of
   sbg_search4_shared.
3. With oracle/_ref/sboxgates_gpu built: drop-in runs without either switch, with SBG_LUT_SHARED=1,
   with SBG_LUT_CHAIN=1 and with both, one process per run under the committed seed: the LUT count
   of the last graph written, whether every graph written verifies (sboxgates_b200/graph.py), the
   wall time, and the nodes that took the shared stage and its seconds (from SBG_SHIM_STATS).
   Without a switch the file names (which carry the graph's fingerprint) are compared with
   tests/golden/xml_names.json where it lists the run.

    python scripts/search4_shared_time.py [--n 40 64] [--reps 5] [--timeout 600] [--no-dropin]
"""
import argparse
import glob
import json
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
from sboxgates_b200 import graph as G  # noqa: E402
from sboxgates_b200.rng import Xorshift1024  # noqa: E402

RUNS = [("des_s1.txt", ["-l", "-o", "0"], "seed1"), ("des_s1.txt", ["-l", "-o", "0"], "seed2"),
        ("crypto1_fc.txt", ["-l"], "seed1"), ("crypto1_fc.txt", ["-l"], "seed2"),
        ("rijndael.txt", ["-l", "-o", "0"], "seed1"), ("sodark.txt", ["-l", "-o", "0"], "seed1")]
CONFIGS = [("plain", {}), ("shared", {"SBG_LUT_SHARED": "1"}), ("chain", {"SBG_LUT_CHAIN": "1"}),
           ("both", {"SBG_LUT_SHARED": "1", "SBG_LUT_CHAIN": "1"})]


def bench_states(eng, ns, reps, seed):
    print("1. bench.py's states: sbg_search5, sbg_search4_shared and the counting sbg_enum4_shared "
          "(ms)")
    print("%4s %5s | %9s | %9s %10s %5s %14s | %10s %12s" % (
        "n", "mask", "search5", "shared", "feasible", "found", "key", "enum4", "total"),
        flush=True)
    for n in ns:
        for st in bench.build_batch(n, 4, seed):
            eng.load(st["tables"], st["target"], st["mask"], st["inbits"])
            o = st["order5"]
            ms5, _ = timed(lambda: eng.search5(o), reps)
            mss, rs = timed(lambda: eng.search4_shared(o), reps)
            mse, e = timed(lambda: eng.enumerate4_shared(o, 0), reps)
            positions = sum(bin(int(w)).count("1") for w in st["mask"])
            print("%4d %5d | %9.3f | %9.3f %10d %5d %14s | %10.3f %12d" % (
                n, positions, ms5, mss, e.feasible, rs.found, hex(rs.key) if rs.found else "-",
                mse, e.total), flush=True)


def recorded_calls(eng):
    calls = []
    for path in sorted(glob.glob(os.path.join(S.GOLDEN, "run_*.bin"))):
        for rec in S.read_records(path):
            if rec.which == 5 and not rec.found:
                calls.append(rec)
    found, ms = 0, []
    for rec in calls:
        order = sb.shuffled_order(Xorshift1024.from_state(rec.rng_s, rec.rng_p))
        eng.load(rec.tables, rec.target, rec.mask, rec.inbits_list())
        eng.search5(order)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = eng.search4_shared(order)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        found += int(res.found)
    print("2. recorded unmatched search_5lut calls: %d, with a shared-input circuit: %d; "
          "sbg_search4_shared per call median %.3f ms, max %.3f ms" % (
              len(calls), found, float(np.median(ms)), max(ms)), flush=True)


def _one(exe, sbox, cli, seed, env_extra, timeout):
    env = dict(os.environ, SBG_SEEDFILE=os.path.join(S.GOLDEN, seed + ".bin"), SBG_SHIM_STATS="1")
    env.update(env_extra)
    sb_tt, _ = G.load_sbox(os.path.join(S.REF_DIR, "sboxes", sbox))
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.time()
        try:
            res = subprocess.run([exe] + cli + [os.path.join(S.REF_DIR, "sboxes", sbox)], cwd=tmp,
                                 env=env, capture_output=True, text=True, timeout=timeout)
        except subprocess.TimeoutExpired:
            return dict(luts="timeout", wall=time.time() - t0)
        wall = time.time() - t0
        files = sorted(glob.glob(os.path.join(tmp, "*.xml")))
        if res.returncode != 0 or not files:
            return dict(luts="rc %d" % res.returncode, wall=wall)
        ok = True
        for f in files:
            try:
                ok &= len(G.verify_graph(G.load_graph(f), sb_tt)) > 0
            except G.GraphError:
                ok = False
        m = re.search(r"shared-input stage: \d+ calls ([0-9.]+) s, (\d+) nodes", res.stderr)
        return dict(luts=str(int(os.path.basename(files[-1]).split("-")[1])), wall=wall,
                    verified=ok, nodes=m.group(2) if m else "-", secs=m.group(1) if m else "-",
                    names=[os.path.basename(f) for f in files])


def dropin(timeout):
    exe = os.path.join(S.REF_DIR, "sboxgates_gpu")
    if not os.path.exists(exe):
        print("3. drop-in: oracle/_ref/sboxgates_gpu not built")
        return
    names = json.load(open(os.path.join(S.GOLDEN, "xml_names.json")))
    print("3. drop-in runs: per configuration LUTs of the last graph / every graph verified / wall s;"
          " shared-stage nodes and seconds")
    for sbox, cli, seed in RUNS:
        cols = []
        for name, extra in CONFIGS:
            r = _one(exe, sbox, cli, seed, extra, timeout)
            col = "%s %s/%s/%.2f" % (name, r["luts"], "ok" if r.get("verified") else "NO",
                                     r["wall"])
            if "SBG_LUT_SHARED" in extra:
                col += " [%s nodes %s s]" % (r.get("nodes"), r.get("secs"))
            if name == "plain":
                want = names.get("%s %s %s" % (sbox, " ".join(cli), seed))
                col += " names %s" % ("-" if want is None else
                                      "same" if want == r.get("names") else "DIFFER")
            cols.append(col)
        print("%-14s %-9s %5s | %s" % (sbox, " ".join(cli), seed, " | ".join(cols)), flush=True)


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
