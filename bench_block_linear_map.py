#!/usr/bin/env python
"""bench_block_linear_map.py -- block linear maps (SURVEY 8f-1): BlockMatMul1DExec::mul's non-iterative branches
(src/matmul.cpp:1782-1868 native, 1869-1974 bad dimension), a GF(p)-linear map on slots of degree d: d0 hoisted rotations,
d0*d1 constant blocks, d1 outer rotations (and, in a bad dimension, a second set of blocks whose sum is rotated once more).

Compares, alternating in one process on the same inputs:
  fused     hb_block_linear_map: k_ks_hoist + k_bsgs_mac per chunk of inner amounts, then the mod-down, digits and k_ks_giant
  seeded    the fused call with every a_i held as its PRG seed and regenerated on each call
  abi       the existing entry points: d0 hb_automorph_keyswitch_digits (hb_add_primes_and_scale for k0 = 1) into full
            rotations, then one extended-form hb_bsgs_linear_map per set (and one for the final rotation)
  steps     HElib's step-by-step engine path: the same rotations, then per outer amount MUL/ADD over the blocks,
            hb_automorph, hb_scale_down, hb_break_into_digits, hb_keyswitch_digits, hb_add_primes_and_scale and ADD
on config 5's ring (m = 21845, p = 2, d = 16) with its three dimensions' real amounts, and config 3's ring (m = 2^17,
p = 257) with synthetic 16 x 16 amounts, B = 1 and 8 ciphertexts.  The four outputs are compared bit for bit.  Reports
the medians with their ranges, the algorithmic GB/s of the fused call's kernels (hb_ctx_profile), the device memory the
engine holds and the card.  1 GPU; writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_bsgs import composed  # noqa: E402

RINGS = {
    "cfg5": {"name": "m=21845 p=2 bits=580 c=2 (thin bootstrapping)", "m": 21845, "p": 2, "bits": 580, "c": 2},
    "cfg3": {"name": "bgv m=2^17 p=257 bits=1500 c=3", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3},
}
# (label, generator, D, bad): config 5's dimensions (orders 16, 4 and a bad 16); config 3's is synthetic, D = d = 16
DIMS = {
    "cfg5": [("dim0", 8996, 16, False), ("dim1", 17477, 4, False), ("dim2", 21591, 16, True)],
    "cfg3": [("synthetic", 5, 16, False)],
}
D_SLOT = 16   # the slot degree d used for the Frobenius amounts p^j (config 5's d; config 3's synthetic inner size)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def amounts(m, p, gen, D, d):
    """BlockMatMul1DExec's strategy: +1 (D >= d) hoists the dimension's rotations and rotates by the Frobenius p^j;
    -1 the other way round.  kfinal = genToPow(dim, -D) for a bad dimension."""
    rot = [pow(gen, i, m) for i in range(D)]
    frob = [pow(p, j, m) for j in range(d)]
    k0, k1 = (rot, frob) if D >= d else (frob, rot)
    return k0, k1, pow(gen, -D, m)


def rotations(E, digits, S, C0, C1, k0, EA0, EB0, R0, R1):
    """r_i = BasicAutomorphPrecon::automorph(k0[i]) for every item, into R0/R1[item][i], over S | special."""
    Sp = sorted(S + E.special)
    for i, k in enumerate(k0):
        o0, o1 = [r[i] for r in R0], [r[i] for r in R1]
        if k == 1:
            E.zero_rows(o0 + o1, Sp)
            E.pointwise("copy", o0 + o1, C0 + C1, S)
            E.add_primes_and_scale(o0 + o1, S, E.special)
        else:
            E.automorph_keyswitch_digits(digits, S, C0, k, EA0[i], EB0[i], o0, o1)


def _t(cs):
    """consts[i][j] (HElib's multiplier[i*d1 + j]) as the BSGS layout [giant j][baby i]"""
    return [list(col) for col in zip(*cs)]


def existing_abi(E, digits, S, C0, C1, k0, EA0, EB0, k1, EA1, EB1, cs, A0, A1, p, cs1=None, kf=1, EAf=None, EBf=None,
                 R0=None, R1=None, Y0=None, Y1=None, one=None):
    """The block map through the existing entry points: full rotations, then extended-form hb_bsgs_linear_map."""
    rotations(E, digits, S, C0, C1, k0, EA0, EB0, R0, R1)
    E.bsgs_linear_map(R0, R1, S, k1, _t(cs), EA1, EB1, A0, A1, extended=True, ptxt_space=p)
    if cs1 is not None:
        E.bsgs_linear_map(R0, R1, S, k1, _t(cs1), EA1, EB1, Y0, Y1, extended=True, ptxt_space=p)
        E.bsgs_linear_map([[y] for y in Y0], [[y] for y in Y1], S, [kf], [[one]], [EAf], [EBf], A0, A1, extended=True,
                          ptxt_space=p, accumulate=True)


def step_by_step(E, digits, S, C0, C1, k0, EA0, EB0, k1, EA1, EB1, cs, A0, A1, p, cs1=None, kf=1, EAf=None, EBf=None,
                 R0=None, R1=None, Y0=None, Y1=None, one=None, tmp=None, Z0=None, Z1=None):
    """HElib's loop through single engine steps: the rotations, then per outer amount MulAdd and smartAutomorph."""
    Sp = sorted(S + E.special)
    rotations(E, digits, S, C0, C1, k0, EA0, EB0, R0, R1)
    composed(E, R0, R1, S, k1, _t(cs), EA1, EB1, A0, A1, 1, p, tmp=tmp)
    if cs1 is not None:
        composed(E, R0, R1, S, k1, _t(cs1), EA1, EB1, Y0, Y1, 1, p, tmp=tmp)
        composed(E, [[y] for y in Y0], [[y] for y in Y1], S, [kf], [[one]], [EAf], [EBf], Z0, Z1, 1, p, tmp=tmp)
        E.pointwise("add", A0 + A1, Z0 + Z1, Sp)


def run_ring(key, Bs, runs, target_s):
    import numpy as np
    import torch
    from helib_b200 import Chain, Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"])
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, device=0)
    E.set_stream(torch.cuda.current_stream().cuda_stream)
    p = R["p"]
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, B, n = len(ch.digits), max(Bs), D_SLOT
    C0, C1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.randomize(C0 + C1, S, 1)
    DG = E.break_into_digits(C1, S)   # the digits of c1 over S, as the ciphertext's hoisting precomputes them
    CS = [[E.poly() for _ in range(n)] for _ in range(n)]
    CS1 = [[E.poly() for _ in range(n)] for _ in range(n)]
    E.randomize([x for r in CS + CS1 for x in r], Sp, 2)
    one = E.poly(np.ones((E.np, E.N), dtype=np.uint64), Sp)
    out = []
    for label, gen, D, bad in DIMS[key]:
        k0, k1, kf = amounts(ch.m, p, gen, D, n)
        n0, n1 = len(k0), len(k1)
        cs, cs1 = [r[:n1] for r in CS[:n0]], ([r[:n1] for r in CS1[:n0]] if bad else None)
        # one matrix per amount, for s(X^k) -> s (none where k = 1): a_i expanded, and as its seed
        def mats(ks, seed):
            EB = [None if k == 1 else [E.poly() for _ in range(nd)] for k in ks]
            EA = [None if k == 1 else [E.poly() for _ in range(nd)] for k in ks]
            SA = [None if k == 1 else E.seeded(nd, Sp, seed + j) for j, k in enumerate(ks)]
            for j, k in enumerate(ks):
                if k != 1:
                    E.randomize(EB[j], Sp, seed + 500 + j)
                    E.randomize(EA[j], Sp, seed + j)
            return EA, EB, SA
        EA0, EB0, SA0 = mats(k0, 1000)
        EA1, EB1, SA1 = mats(k1, 2000)
        EAf, EBf, SAf = mats([kf], 3000) if bad else ([None], [None], [None])
        for b in Bs:
            dg = DG[:b]
            c0, c1 = C0[:b], C1[:b]
            outs = {f: ([E.poly() for _ in range(b)], [E.poly() for _ in range(b)]) for f in ("fused", "seeded", "abi", "steps")}
            R0 = [[E.poly() for _ in range(n0)] for _ in range(b)]
            R1 = [[E.poly() for _ in range(n0)] for _ in range(b)]
            Y0, Y1, Z0, Z1 = ([E.poly() for _ in range(b)] for _ in range(4))
            tmp = [[E.poly() for _ in range(b)] for _ in range(5)]
            extra = dict(cs1=cs1, kf=kf, EAf=EAf[0], EBf=EBf[0]) if bad else {}
            forms = {
                "fused": lambda: E.block_linear_map(dg, S, c0, c1, k0, EA0, EB0, k1, EA1, EB1, cs, *outs["fused"], consts1=cs1,
                                                    kfinal=kf, evkf_a=EAf[0], evkf_b=EBf[0], ptxt_space=p),
                "seeded": lambda: E.block_linear_map(dg, S, c0, c1, k0, SA0, EB0, k1, SA1, EB1, cs, *outs["seeded"], consts1=cs1,
                                                     kfinal=kf, evkf_a=SAf[0], evkf_b=EBf[0], ptxt_space=p),
                "abi": lambda: existing_abi(E, dg, S, c0, c1, k0, EA0, EB0, k1, EA1, EB1, cs, *outs["abi"], p, R0=R0, R1=R1,
                                            Y0=Y0, Y1=Y1, one=one, **extra),
                "steps": lambda: step_by_step(E, dg, S, c0, c1, k0, EA0, EB0, k1, EA1, EB1, cs, *outs["steps"], p, R0=R0, R1=R1,
                                              Y0=Y0, Y1=Y1, one=one, tmp=tmp, Z0=Z0, Z1=Z1, **extra),
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
            got = {f: [x.download(Sp)[Sp] for x in P[0] + P[1]] for f, P in outs.items()}
            identical = all(all(np.array_equal(x, y) for x, y in zip(got["fused"], got[f])) for f in ("seeded", "abi", "steps"))
            E.profile(True)
            forms["fused"]()
            prof = {r["kernel"]: r for r in E.profile_results()}
            E.profile(False)
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            kern = {}
            for kname in ("k_ks_hoist", "k_bsgs_mac", "k_ks_giant"):
                k = prof.get(kname, {"ms": 0.0, "bytes": 0, "launches": 0})
                kern[kname] = {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                               "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None}
            rec = {"ring": key, "ring_name": R["name"], "m": ch.m, "phim": E.N, "rows": len(Sp), "digits": nd, "dim": label,
                   "D": D, "d0": n0, "d1": n1, "bad": bad, "items": b, "device_GB": E.stats()["device_bytes"] / 1e9,
                   "ms": {f: [round(x, 4) for x in v] for f, v in ms.items()},
                   "median_ms": {f: round(v, 4) for f, v in med.items()},
                   "range_ms": {f: [round(min(v), 4), round(max(v), 4)] for f, v in ms.items()},
                   "speedup_fused_vs_steps": med["steps"] / med["fused"], "speedup_fused_vs_abi": med["abi"] / med["fused"],
                   "kernels": kern, "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
            del R0, R1, tmp
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg5,cfg3")
    ap.add_argument("--items", default="1,8")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.25, help="seconds of work per timed run")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_block_linear_map.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.items.split(",")], a.runs, a.window)
    print(json.dumps({"metric": "block_linear_map", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_than_steps_everywhere": all(r["speedup_fused_vs_steps"] > 1 for r in recs),
                      "fused_faster_than_abi_everywhere": all(r["speedup_fused_vs_abi"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
