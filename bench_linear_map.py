#!/usr/bin/env python
"""bench_linear_map.py -- hoisted linear maps (SURVEY 8f-1): sum_j C_j * automorph(k_j) of one ciphertext over one digit
decomposition, the loop body of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252).

Compares, alternating in one process on the same inputs:
  fused     hb_hoisted_linear_map: one k_ks_linmap pass per group of up to 64 amounts
  composed  per amount hb_automorph_keyswitch_digits + hb_pointwise MUL + ADD (what a caller builds without the fused call)
  seeded    the fused call with every a_i held as its PRG seed and regenerated on each call
on config 5's ring (m = 21845, the thin-bootstrapping chain of bench_general_m.py) and config 3's (m = 2^17, 3 digits),
D = 16 and 64 amounts with one matrix each, B = 1 and 8 ciphertexts.  The three outputs are compared bit for bit.
Reports linear maps/s, amounts/s, the algorithmic GB/s of k_ks_linmap (hb_ctx_profile) and the card.  1 GPU; writes
nothing to disk."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RINGS = {
    "cfg5": {"name": "m=21845 p=2 bits=580 c=2 (thin bootstrapping)", "m": 21845, "p": 2, "bits": 580, "c": 2},
    "cfg3": {"name": "bgv m=2^17 p=257 bits=1500 c=3", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3},
}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def composed(E, digs, S, C0, ks, CS, EA, EB, A0, A1, T0, T1):
    Sp = sorted(S + E.special)
    for j, k in enumerate(ks):
        o0, o1 = (A0, A1) if j == 0 else (T0, T1)
        E.automorph_keyswitch_digits(digs, S, C0, k, EA[j], EB[j], o0, o1)
        E.pointwise("mul", o0 + o1, [CS[j]] * (2 * len(o0)), Sp)
        if j:
            E.pointwise("add", A0 + A1, T0 + T1, Sp)


def run_ring(key, Ds, Bs, runs, target_s):
    import numpy as np
    import torch
    from helib_b200 import Chain, Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"])
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, device=0)
    E.set_stream(torch.cuda.current_stream().cuda_stream)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, D, B = len(ch.digits), max(Ds), max(Bs)
    ks = [t for t in range(3, ch.m) if math.gcd(t, ch.m) == 1][:D]
    C0, C1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.randomize(C0 + C1, S, 1)
    digs = E.break_into_digits(C1, S)
    CS = [E.poly() for _ in range(D)]
    E.randomize(CS, Sp, 2)
    EB = [[E.poly() for _ in range(nd)] for _ in range(D)]
    E.randomize([x for m in EB for x in m], Sp, 3)
    EA = [[E.poly() for _ in range(nd)] for _ in range(D)]
    for j in range(D):
        E.randomize(EA[j], Sp, 1000 + j)
    SA = [E.seeded(nd, Sp, 1000 + j) for j in range(D)]
    A0, A1, R0, R1, T0, T1, Z0, Z1 = ([E.poly() for _ in range(B)] for _ in range(8))
    out = []
    for d in Ds:
        for b in Bs:
            forms = {
                "fused": lambda: E.hoisted_linear_map(digs[:b], S, C0[:b], None, ks[:d], CS[:d], EA[:d], EB[:d], A0[:b], A1[:b]),
                "composed": lambda: composed(E, digs[:b], S, C0[:b], ks[:d], CS[:d], EA[:d], EB[:d], R0[:b], R1[:b], T0[:b], T1[:b]),
                "seeded": lambda: E.hoisted_linear_map(digs[:b], S, C0[:b], None, ks[:d], CS[:d], SA[:d], EB[:d], Z0[:b], Z1[:b]),
            }
            steps = {}
            for f, fn in forms.items():   # warm every shape, then size the timed window
                fn()
                torch.cuda.synchronize()
                E.mark_begin(); fn(); ms = E.mark_end()
                steps[f] = max(3, min(200, int(target_s * 1e3 / max(ms, 1e-3))))
            ms = {f: [] for f in forms}
            for _ in range(runs):
                for f, fn in forms.items():
                    E.mark_begin()
                    for _ in range(steps[f]):
                        fn()
                    ms[f].append(E.mark_end() / steps[f])
            got = {f: [x.download(Sp)[Sp] for x in P] for f, P in (("fused", A0[:b] + A1[:b]), ("composed", R0[:b] + R1[:b]), ("seeded", Z0[:b] + Z1[:b]))}
            identical = all(np.array_equal(x, y) for x, y in zip(got["fused"], got["composed"])) and \
                all(np.array_equal(x, y) for x, y in zip(got["fused"], got["seeded"]))
            E.profile(True)
            forms["fused"]()
            prof = {r["kernel"]: r for r in E.profile_results()}
            E.profile(False)
            k = prof.get("k_ks_linmap", {"ms": 0.0, "bytes": 0, "launches": 0})
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            rec = {"ring": key, "ring_name": R["name"], "m": ch.m, "phim": E.N, "rows": len(Sp), "digits": nd, "amounts": d, "items": b,
                   "ms": {f: [round(x, 4) for x in v] for f, v in ms.items()},
                   "maps_per_s": {f: b / (med[f] / 1e3) for f in forms},
                   "amounts_per_s": {f: b * d / (med[f] / 1e3) for f in forms},
                   "speedup_fused_vs_composed": med["composed"] / med["fused"],
                   "k_ks_linmap": {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                                   "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None},
                   "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg5,cfg3")
    ap.add_argument("--amounts", default="16,64")
    ap.add_argument("--items", default="1,8")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.25, help="seconds of work per timed run")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_linear_map.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.amounts.split(",")], [int(x) for x in a.items.split(",")], a.runs, a.window)
    print(json.dumps({"metric": "hoisted_linear_map", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_everywhere": all(r["speedup_fused_vs_composed"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
