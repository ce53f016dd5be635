#!/usr/bin/env python3
"""CPU: which window forms a full phase-1 sweep of search_7lut's shifted-window filter goes through.

  python scripts/filter_windows.py [n] [excluded input bits, e.g. 0,3]

Enumerates the (prefix, chunk of 32 (e,f) pairs) items the way k_filter7_pm does for a sweep that
runs to the end (4-gate prefixes over the allowed gates; prefixes that hold an excluded gate are
stepped over) and classifies each chunk's windows by the candidate gates they span:
quad (<= 7: four parts per register), packed (<= 15: two parts) or single (up to 31: one part).
Two rules for where a chunk's first window starts are compared:
  per prefix -- at the prefix's last gate + 3 (the smallest g any of its pairs can take);
  per chunk  -- at the smallest f + 1 over the chunk's live lanes (what the kernel does).
Counts only: no timing, no GPU.  With a -DSBG_COUNT_FILTER build of the library the kernel prints
the same window counts per launch (the "windows", "packed" and "quad" fields of its F1 line)."""
import sys
from math import comb


def classify(left):
    return "quad" if left <= 7 else "packed" if left <= 15 else "single"


def windows(base, n):
    """Classes of the 31-gate windows from `base` on (base, base + 31, ... < n)."""
    return [classify(n - b) for b in range(base, n, 31)]


def sweep(n, inbits=()):
    excl = set(b for b in inbits if b < 8)
    allowed = [g for g in range(n) if g not in excl]
    forms = ("quad", "packed", "single")
    out = {rule: {"chunks": 0, "first": dict.fromkeys(forms, 0), "windows": dict.fromkeys(forms, 0)}
           for rule in ("per_prefix", "per_chunk")}
    for last in range(3, n - 3):   # prefix (a, b, c, last): three more gates above it
        if last in excl:
            continue
        prefixes = comb(sum(1 for g in allowed if g < last), 3)
        if prefixes == 0:
            continue
        r = n - last - 2           # e, f among last+1 .. n-2
        pairs = [(i, j) for i in range(r - 1) for j in range(i + 1, r)]
        for c0 in range(0, len(pairs), 32):
            live = [last + 1 + j for i, j in pairs[c0:c0 + 32]
                    if last + 1 + i not in excl and last + 1 + j not in excl]
            for rule, base in (("per_prefix", last + 3),
                               ("per_chunk", min(live) + 1 if live else None)):
                rec = out[rule]
                rec["chunks"] += prefixes
                if base is None:   # no live lane: the kernel skips the chunk
                    continue
                ws = windows(base, n)
                rec["first"][ws[0]] += prefixes
                for w in ws:
                    rec["windows"][w] += prefixes
    return out


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    inbits = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 and sys.argv[2] else []
    res = sweep(n, inbits)
    print("n = %d, excluded input bits %s: %d chunks per sweep"
          % (n, inbits or "none", res["per_chunk"]["chunks"]))
    for rule, rec in res.items():
        tot = sum(rec["first"].values())
        print("  %-10s chunks by first window: %s   windows: %s" % (
            rule, "  ".join("%s %.1f %%" % (k, 100.0 * v / max(tot, 1)) for k, v in rec["first"].items()),
            "  ".join("%s %d" % kv for kv in rec["windows"].items())))


if __name__ == "__main__":
    main()
