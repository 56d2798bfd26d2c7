#!/usr/bin/env python
"""bench_bsgs.py -- BSGS linear maps (SURVEY 8f-1): the giant-step phase of MatMul1DExec::mul's non-iterative
baby-step/giant-step branches (src/matmul.cpp:1022-1057 native, 1097-1142 bad dimension), D diagonals over g = ceil(sqrt(D))
baby steps and h = ceil(D/g) giant steps.

Compares, alternating in one process on the same inputs:
  fused     hb_bsgs_linear_map: per group of giant steps one k_bsgs_mac pass, the batched mod-down and digits, one k_ks_giant
  composed  per giant step MUL/ADD over the baby steps, hb_automorph, [hb_scale_down], hb_break_into_digits,
            hb_keyswitch_digits, hb_add_primes_and_scale, ADD (what a caller builds without the fused call)
  seeded    the fused call with every a_i held as its PRG seed and regenerated on each call
on config 2's ring (CKKS m = 2^17, native form) and config 5's (m = 21845, p = 2, the extended form of a bad dimension:
2g baby steps over S | special), D = 256 and 1024, B = 1 and 8 ciphertexts.  The three outputs are compared bit for bit.
Reports the medians, the algorithmic GB/s of both kernels (hb_ctx_profile), the device memory the engine holds and the
card.  1 GPU; writes nothing to disk."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RINGS = {
    "cfg2": {"name": "ckks m=2^17 bits=1190 c=2", "m": 1 << 17, "p": -1, "bits": 1190, "c": 2, "extended": 0},
    "cfg5": {"name": "m=21845 p=2 bits=580 c=2 (thin bootstrapping), extended form", "m": 21845, "p": 2, "bits": 580, "c": 2, "extended": 1},
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


def composed(E, B0, B1, S, ks, CS, EA, EB, A0, A1, extended, p, scal=None, tmp=None):
    """The giant steps through the engine's single steps: per giant step MUL/ADD over the baby steps, hb_automorph,
    [hb_scale_down], hb_break_into_digits, hb_keyswitch_digits, hb_add_primes_and_scale, ADD.  tmp: five lists of
    len(B0) scratch Polys (allocated if None)."""
    Sp = sorted(S + E.special)
    R = Sp if extended else S
    nit = len(B0)
    x0, x1, y0, y1, t = tmp if tmp is not None else ([E.poly() for _ in range(nit)] for _ in range(5))
    E.zero_rows(A0 + A1, Sp)
    for g, k in enumerate(ks):
        E.zero_rows(x0 + x1, R)
        for j, c in enumerate(CS[g]):
            if c is None:
                continue
            for xs, bs in ((x0, B0), (x1, B1)):
                E.pointwise("copy", t, [b[j] for b in bs], R)
                E.pointwise("mul", t, [c] * nit, R)
                E.pointwise("add", xs, t, R)
        if k == 1:
            if not extended:
                E.add_primes_and_scale(x0 + x1, S, E.special)
            E.pointwise("add", A0 + A1, x0 + x1, Sp)
            continue
        E.automorph(y0 + y1, x0 + x1, R, k)
        if extended:
            E.scale_down(y0 + y1, Sp, S, p)
        if scal is not None and scal[g] != 1:
            E.scale_rows(y0 + y1, S, [scal[g] % E.primes[i] for i in S])
        digs = E.break_into_digits(y1, S)
        E.add_primes_and_scale(y0, S, E.special)
        E.zero_rows(y1, Sp)
        E.keyswitch_digits(digs, Sp, EA[g], EB[g], y0, y1)
        E.pointwise("add", A0 + A1, y0 + y1, Sp)


def gen_of(m):
    return next(t for t in range(2, m) if math.gcd(t, m) == 1 and pow(t, 2, m) != 1)


def run_ring(key, Ds, Bs, runs, target_s):
    import numpy as np
    import torch
    from helib_b200 import Chain, Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"])
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, device=0)
    E.set_stream(torch.cuda.current_stream().cuda_stream)
    ext, p = R["extended"], (1 if R["p"] == -1 else R["p"])
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    rows = Sp if ext else S
    nd, B = len(ch.digits), max(Bs)
    gmax = max(math.isqrt(d - 1) + 1 for d in Ds)
    hmax = max(-(-d // (math.isqrt(d - 1) + 1)) for d in Ds)
    nbmax = gmax * (2 if ext else 1)
    B0 = [[E.poly() for _ in range(nbmax)] for _ in range(B)]
    B1 = [[E.poly() for _ in range(nbmax)] for _ in range(B)]
    E.randomize([x for it in B0 + B1 for x in it], rows, 1)
    CS = [[E.poly() for _ in range(nbmax)] for _ in range(hmax)]
    E.randomize([x for r in CS for x in r], rows, 2)
    EB = [[E.poly() for _ in range(nd)] for _ in range(hmax)]
    E.randomize([x for m in EB for x in m], Sp, 3)
    EA = [[E.poly() for _ in range(nd)] for _ in range(hmax)]
    for j in range(hmax):
        E.randomize(EA[j], Sp, 1000 + j)
    SA = [E.seeded(nd, Sp, 1000 + j) for j in range(hmax)]
    A0, A1, R0, R1, Z0, Z1 = ([E.poly() for _ in range(B)] for _ in range(6))
    tmp = [[E.poly() for _ in range(B)] for _ in range(5)]
    gen = gen_of(ch.m)
    out = []
    for d in Ds:
        g = math.isqrt(d - 1) + 1
        h = -(-d // g)
        nb = g * (2 if ext else 1)
        ks = [pow(gen, g * t, ch.m) for t in range(h)]
        # diagonal i = j + g*k of giant step k; past D there is none (MulAdd is not called)
        cs = [[CS[k][j] if (j % g) + g * k < d else None for j in range(nb)] for k in range(h)]
        for b in Bs:
            b0, b1 = [x[:nb] for x in B0[:b]], [x[:nb] for x in B1[:b]]
            forms = {
                "fused": lambda: E.bsgs_linear_map(b0, b1, S, ks, cs, EA[:h], EB[:h], A0[:b], A1[:b], extended=ext, ptxt_space=p),
                "composed": lambda: composed(E, b0, b1, S, ks, cs, EA[:h], EB[:h], R0[:b], R1[:b], ext, p, tmp=[x[:b] for x in tmp]),
                "seeded": lambda: E.bsgs_linear_map(b0, b1, S, ks, cs, SA[:h], EB[:h], Z0[:b], Z1[:b], extended=ext, ptxt_space=p),
            }
            steps = {}
            for f, fn in forms.items():   # warm every shape, then size the timed window
                fn()
                torch.cuda.synchronize()
                E.mark_begin(); fn(); ms = E.mark_end()
                steps[f] = max(3, min(100, int(target_s * 1e3 / max(ms, 1e-3))))
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
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            kern = {}
            for kname in ("k_bsgs_mac", "k_ks_giant"):
                k = prof.get(kname, {"ms": 0.0, "bytes": 0, "launches": 0})
                kern[kname] = {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                               "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None}
            rec = {"ring": key, "ring_name": R["name"], "m": ch.m, "phim": E.N, "rows": len(Sp), "digits": nd, "extended": ext,
                   "D": d, "g": g, "h": h, "items": b, "device_GB": E.stats()["device_bytes"] / 1e9,
                   "ms": {f: [round(x, 4) for x in v] for f, v in ms.items()},
                   "median_ms": {f: round(v, 4) for f, v in med.items()},
                   "speedup_fused_vs_composed": med["composed"] / med["fused"],
                   "kernels": kern, "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg2,cfg5")
    ap.add_argument("--dims", default="256,1024")
    ap.add_argument("--items", default="1,8")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.25, help="seconds of work per timed run")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_bsgs.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.dims.split(",")], [int(x) for x in a.items.split(",")], a.runs, a.window)
    print(json.dumps({"metric": "bsgs_linear_map", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_everywhere": all(r["speedup_fused_vs_composed"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
