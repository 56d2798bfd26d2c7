#!/usr/bin/env python
"""bench_inner_product.py -- encrypted inner products: innerProduct (src/Ctxt.cpp:2878-2893), B vectors of n pairs each,
every operand over S_in and the common set S one prime lower (the pairs' rescale drops a prime).

Compares, alternating in one process on the same inputs:
  fused           hb_inner_product: the lazy scale-down of all parts, one k1_tensor_sum pass, one relinearisation and
                  mod-down per item
  lazy-composed   hb_scale_down of all parts, per pair hb_tensor and three ADDs, then hb_relinearize + hb_scale_down (the
                  same arithmetic through the existing entry points)
  multiply-each   one batched hb_mul_relin_moddown over all n*B pairs, then ADDs (what a caller without innerProduct
                  writes: a key switch per pair)
on config 2's ring (CKKS m = 2^17, 20 + 10 primes) and config 3's (BGV m = 2^17, p = 257, 3 digits), n = 4, 16, 64 and
B = 1, 4.  The operands are consumed (brought to S in place); they are restored from a few pristine pairs by device copies
before every call, outside the timed window.  fused and lazy-composed must be bit-identical; multiply-each relinearises
every pair, so it is only timed.  Reports medians and ranges over --runs, inner products/s and pairs/s, k1_tensor_sum's
algorithmic GB/s (hb_ctx_profile, a separate pass) and the card with its power limit.  1 GPU; writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RINGS = {
    "cfg2": {"name": "ckks m=2^17 bits=1190 c=2", "m": 1 << 17, "p": -1, "bits": 1190, "c": 2},
    "cfg3": {"name": "bgv m=2^17 p=257 bits=1500 c=3", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3},
}
PRISTINE = 4   # distinct random pairs the operands are restored from


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def run_ring(key, ns, Bs, runs):
    import torch
    from helib_b200 import Chain
    from helib_b200.engine import Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"], lib=None)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special)
    p = 1 if R["p"] == -1 else R["p"]
    S_in = ch.ctxt
    S = ch.ctxt[:-1]
    Sp = sorted(S + ch.special)
    nd = len(ch.digits)
    EB = [E.poly() for _ in range(nd)]
    E.randomize(EB, Sp, 3)
    EA = [E.poly() for _ in range(nd)]
    E.randomize(EA, Sp, 1000)
    P = [[E.poly() for _ in range(4)] for _ in range(PRISTINE)]
    E.randomize([x for pr in P for x in pr], S_in, 7)
    nmax = max(ns) * max(Bs)
    W = [[E.poly() for _ in range(4)] for _ in range(nmax)]     # the operands of one call, restored before each
    O0, O1, C0, C1, C2, M0, M1 = ([E.poly() for _ in range(max(Bs))] for _ in range(7))
    T = [[E.poly() for _ in range(max(Bs))] for _ in range(3)]
    out = []
    for n in ns:
        for b in Bs:
            w = W[:n * b]

            def restore():
                for k in range(4):
                    E.pointwise("copy", [pr[k] for pr in w], [P[i % PRISTINE][k] for i in range(n * b)], S_in)

            parts = [[[w[t * n + j][k] for j in range(n)] for t in range(b)] for k in range(4)]

            def fused():
                E.inner_product(*parts, S_in, S, p, EA, EB, O0[:b], O1[:b], moddown=True)

            def composed():
                E.scale_down([x for pr in w for x in pr], S_in, S, p)
                acc = (C0[:b], C1[:b], C2[:b])
                E.tensor(*([w[t * n][k] for t in range(b)] for k in range(4)), *acc, S)
                for j in range(1, n):
                    E.tensor(*([w[t * n + j][k] for t in range(b)] for k in range(4)), *(x[:b] for x in T), S)
                    for k in range(3):
                        E.pointwise("add", acc[k], T[k][:b], S)
                E.relinearize(*acc, S, EA, EB)
                E.scale_down(C0[:b] + C1[:b], Sp, S, p)

            def each():
                E.mul_relin_moddown(*([pr[k] for pr in w] for k in range(4)), S_in, S, p, EA, EB)
                for t in range(b):   # the results sit in (a0, a1) of every pair
                    E.pointwise("copy", [M0[t], M1[t]], [w[t * n][0], w[t * n][1]], S)
                for j in range(1, n):
                    E.pointwise("add", M0[:b] + M1[:b], [w[t * n + j][0] for t in range(b)] + [w[t * n + j][1] for t in range(b)], S)

            forms = {"fused": fused, "lazy-composed": composed, "multiply-each": each}

            def timed(fn):
                restore()
                torch.cuda.synchronize()
                E.mark_begin()
                fn()
                return E.mark_end()

            for fn in forms.values():   # warm every shape (first-use allocations, conversion tables)
                timed(fn)
            ms = {f: [] for f in forms}
            for _ in range(runs):
                for f, fn in forms.items():
                    ms[f].append(timed(fn))
            restore(); fused()
            restore(); composed()
            identical = all(np.array_equal(x.download(S)[S], y.download(S)[S]) for x, y in zip(O0[:b] + O1[:b], C0[:b] + C1[:b]))
            restore()
            torch.cuda.synchronize()
            E.profile(True)
            fused()
            prof = {r["kernel"]: r for r in E.profile_results()}
            E.profile(False)
            k = prof.get("k1_tensor_sum", {"ms": 0.0, "bytes": 0, "launches": 0})
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            rec = {"ring": key, "ring_name": R["name"], "phim": E.N, "ctxt_primes": len(S_in), "special": len(ch.special), "digits": nd,
                   "pairs": n, "items": b, "device_GB": E.stats()["device_bytes"] / 1e9,
                   "ms": {f: [round(x, 4) for x in v] for f, v in ms.items()},
                   "median_ms": {f: round(v, 4) for f, v in med.items()},
                   "range_ms": {f: [round(min(v), 4), round(max(v), 4)] for f, v in ms.items()},
                   "inner_products_per_s": {f: b / (v / 1e3) for f, v in med.items()},
                   "pairs_per_s": {f: n * b / (v / 1e3) for f, v in med.items()},
                   "speedup_fused_vs_lazy_composed": med["lazy-composed"] / med["fused"],
                   "speedup_fused_vs_multiply_each": med["multiply-each"] / med["fused"],
                   "k1_tensor_sum": {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                                     "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None},
                   "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg2,cfg3")
    ap.add_argument("--pairs", default="4,16,64")
    ap.add_argument("--items", default="1,4")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_inner_product.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.pairs.split(",")], [int(x) for x in a.items.split(",")], a.runs)
    print(json.dumps({"metric": "inner_product", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_than_multiply_each_everywhere": all(r["speedup_fused_vs_multiply_each"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
