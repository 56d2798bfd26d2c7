#!/usr/bin/env python
"""bench_square.py -- squaring ciphertexts: Ctxt::square (multiplyBy(*this), src/Ctxt.cpp:1704-1708,1757-1774) of B
ciphertexts, every operand over S_in and the target set S one prime lower (the square's rescale drops a prime).

Compares, alternating in one process on the same inputs:
  fused           hb_square_relin_moddown: the conversion of the two parts, one k1_fwd_blk_square pass (rescale and
                  self-tensor), one relinearisation and mod-down per item
  multiply-copy   hb_mul_relin_moddown(x, copy of x): what a caller without a square writes (the copy is made outside the
                  timed window); it rescales four parts where two would do
  composed        hb_scale_down of the two parts, hb_tensor(x, x) in place, hb_relinearize, hb_scale_down (the same
                  arithmetic through the existing entry points)
on config 2's ring (CKKS m = 2^17, 20 ctxt primes) and config 3's (BGV m = 2^17, p = 257), B = 1, 8, 32.  The operands
are consumed (squared in place); they are restored from a few pristine ciphertexts by device copies before every call,
outside the timed window.  The three outputs must be bit-identical.  Reports medians and ranges over --runs, squares/s,
speed-ups, k1_fwd_blk_square's ms and algorithmic GB/s (hb_ctx_profile, a separate pass) and the card with its power
limit.  1 GPU; writes nothing to disk."""
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
PRISTINE = 4   # distinct random ciphertexts the operands are restored from


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def run_ring(key, Bs, runs):
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
    P = [[E.poly() for _ in range(2)] for _ in range(PRISTINE)]
    E.randomize([x for c in P for x in c], S_in, 7)
    bmax = max(Bs)
    X = [[E.poly() for _ in range(2)] for _ in range(bmax)]     # the operands of one call, restored before each
    Y = [[E.poly() for _ in range(2)] for _ in range(bmax)]     # multiply-copy's second operands
    T2 = [E.poly() for _ in range(bmax)]                        # composed: the s^2 part
    out = []
    for b in Bs:
        x, y = X[:b], Y[:b]

        def restore():
            for k in range(2):
                E.pointwise("copy", [c[k] for c in x], [P[i % PRISTINE][k] for i in range(b)], S_in)
                E.pointwise("copy", [c[k] for c in y], [P[i % PRISTINE][k] for i in range(b)], S_in)

        x0, x1, y0, y1 = [c[0] for c in x], [c[1] for c in x], [c[0] for c in y], [c[1] for c in y]

        def fused():
            E.square_relin_moddown(x0, x1, S_in, S, p, EA, EB)

        def multiply_copy():
            E.mul_relin_moddown(x0, x1, y0, y1, S_in, S, p, EA, EB)

        def composed():
            E.scale_down(x0 + x1, S_in, S, p)
            E.tensor(x0, x1, x0, x1, x0, x1, T2[:b], S)
            E.relinearize(x0, x1, T2[:b], S, EA, EB)
            E.scale_down(x0 + x1, Sp, S, p)

        forms = {"fused": fused, "multiply-copy": multiply_copy, "composed": composed}

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
        res = {}
        for f, fn in forms.items():
            restore()
            fn()
            res[f] = [c.download(S)[S] for c in x0 + x1]
        identical = all(np.array_equal(a, c) for f in ("multiply-copy", "composed") for a, c in zip(res["fused"], res[f]))
        restore()
        torch.cuda.synchronize()
        E.profile(True)
        fused()
        prof = {r["kernel"]: r for r in E.profile_results()}
        E.profile(False)
        k = prof.get("k1_fwd_blk_square", {"ms": 0.0, "bytes": 0, "launches": 0})
        med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
        rec = {"ring": key, "ring_name": R["name"], "phim": E.N, "ctxt_primes": len(S_in), "special": len(ch.special), "digits": nd,
               "items": b, "device_GB": E.stats()["device_bytes"] / 1e9,
               "ms": {f: [round(v, 4) for v in vs] for f, vs in ms.items()},
               "median_ms": {f: round(v, 4) for f, v in med.items()},
               "range_ms": {f: [round(min(v), 4), round(max(v), 4)] for f, v in ms.items()},
               "squares_per_s": {f: b / (v / 1e3) for f, v in med.items()},
               "speedup_fused_vs_multiply_copy": med["multiply-copy"] / med["fused"],
               "speedup_fused_vs_composed": med["composed"] / med["fused"],
               "k1_fwd_blk_square": {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                                     "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None},
               "fused_profile_ms": {n: round(r["ms"], 4) for n, r in prof.items()},
               "bit_identical": identical}
        print(json.dumps(rec), flush=True)
        out.append(rec)
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg2,cfg3")
    ap.add_argument("--items", default="1,8,32")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_square.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.items.split(",")], a.runs)
    print(json.dumps({"metric": "square", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_than_multiply_copy_everywhere": all(r["speedup_fused_vs_multiply_copy"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
