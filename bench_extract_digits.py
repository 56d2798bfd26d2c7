#!/usr/bin/env python
"""bench_extract_digits.py -- digit extraction on the device: the mirror's hb::extractDigits and hb::extractDigitsThin
(src/extractDigits.cpp:70-129, src/recryption.cpp:793-909).

Round i of extractDigits powers digits 0..i-1 (square for p = 2, cube for p = 3, the degree-p digit polynomial through
polyEval otherwise) and then runs the chain tmp -= digits[j]; tmp.divideByP() over them.  Compares, alternating in one
process on the same input:
  fused      the mirror as it stands: each round's chain, and extractDigitsThin's final combination, as one
             hb_ctxt_scaled_sums call (k1_scaled_sums)
  composed   the same calls with the chains and the combination run step by step through the existing entry points
             (addCtxt's mod-up, scalings and adds, divideByP's hb_scale_rows)
on config 5's ring (m = 21845, p = 2: n = 4, 8 and 12 digits), config 3's ring (m = 2^17, p = 257: n = 2 and 3, each
powering a degree-257 polyEval), and extractDigitsThin at one (botHigh, r, e') per ring.  The chains need more levels
than the BASELINE chains hold for the larger n, so each workload's chain length is given in bits.  Each run calls both forms
on fresh outputs, in alternating order.  Reports, per workload, medians and ranges over --runs of the whole call (CUDA events
on the context's stream), of its powerings and of its chains (a second call with the mirror's timers on, which
synchronise at each step), the chains' share of the two, and the fused form's k1_scaled_sums launches, the calls they come
from and their algorithmic GB/s (hb_ctx_profile, a last pass), with the card and its power limit.  The fused and composed
outputs must be bit-identical.  The timing driver (bench_micro/extract_digits_driver.cpp) is compiled into a temporary
directory; 1 GPU; writes nothing to the tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))

#          name                      form     m        p    bits  c  args
WORKLOADS = [
    ("cfg5 n=4",            "digits", 21845, 2, 580, 2, [4]),
    ("cfg5 n=8",            "digits", 21845, 2, 900, 2, [8]),
    ("cfg5 n=12",           "digits", 21845, 2, 1200, 2, [12]),
    ("cfg5 thin 2,3,1",     "thin", 21845, 2, 900, 2, [2, 3, 1]),
    ("cfg3 n=2",            "digits", 1 << 17, 257, 1500, 3, [2]),
    ("cfg3 n=3",            "digits", 1 << 17, 257, 3000, 3, [3]),
    ("cfg3 thin 1,2,1",     "thin", 1 << 17, 257, 2000, 3, [1, 2, 1]),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return out


def build(tmp):
    lib = os.path.join(ROOT, "helib_b200", "libhelib_b200.so")
    if not os.path.exists(lib):
        raise SystemExit("libhelib_b200.so is not built: run build() first")
    exe = os.path.join(tmp, "extract_digits_driver")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "bench_micro", "extract_digits_driver.cpp"), "-o", exe, lib,
                           "-Wl,-rpath," + os.path.dirname(lib)])
    return exe


def stat(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    a = ap.parse_args()
    only = [s.strip() for s in a.only.split(",") if s.strip()]
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        exe = build(tmp)
        for name, form, m, p, bits, c, args in WORKLOADS:
            if only and name not in only:
                continue
            cmd = [exe, form, str(m), str(p), str(bits), str(c)] + [str(x) for x in args] + [str(a.runs)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            line = (r.stdout.strip().splitlines() or ["{}"])[-1]
            try:
                d = json.loads(line)
            except json.JSONDecodeError:
                d = {"error": (r.stdout + r.stderr)[-400:]}
            rec = {"workload": name, "form": form, "m": m, "p": p, "bits": bits, "args": args, "exit": r.returncode}
            if "fused_ms" in d:
                f, k = d["fused_ms"], d["composed_ms"]
                med = statistics.median
                rec.update({
                    "primes": d["primes"],
                    "fused_ms": stat(f), "composed_ms": stat(k),
                    "speedup": round(med(k) / med(f), 3),
                    "fused_power_ms": stat(d["fused_power_ms"]), "composed_power_ms": stat(d["composed_power_ms"]),
                    "fused_chain_ms": stat(d["fused_chain_ms"]), "composed_chain_ms": stat(d["composed_chain_ms"]),
                    "fused_chain_share": round(med(d["fused_chain_ms"]) / (med(d["fused_chain_ms"]) + med(d["fused_power_ms"])), 4),
                    "composed_chain_share": round(med(d["composed_chain_ms"]) / (med(d["composed_chain_ms"]) + med(d["composed_power_ms"])), 4),
                    "chain_calls": d["chain_calls"], "powerings": d["powerings"],
                    "sums_launches": d["sums_launches"],
                    "sums_ms": d["sums_ms"],
                    "sums_GBps": round(d["sums_bytes"] / (d["sums_ms"] * 1e6), 1) if d["sums_ms"] > 0 else None,
                    "identical": d["identical"],
                })
            else:
                rec["error"] = d.get("error", "no result")
            results.append(rec)
            print(json.dumps(rec), flush=True)
    ok = all(r.get("identical") is True for r in results)
    print(json.dumps({"bench": "extract_digits", "card": card(), "runs": a.runs, "all_identical": ok}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
