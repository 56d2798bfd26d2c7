#!/usr/bin/env python
"""bench_full_linear_map.py -- full-matrix linear maps (SURVEY 8f-1): the leaves of MatMulFullExec::rec_mul
(src/matmul.cpp:2141-2148), i.e. one hoisted MatMul1DExec::mul per path through the outer dimensions, all sharing the
leaf dimension's amounts and key-switching matrices and summed into one accumulator.

Compares, alternating in one process on the same leaf inputs:
  fused     hb_full_linear_map_leaves: the leaves' cleanUp and digits batched per chunk, one k_ks_leafmap pass per group
            of amounts summing every leaf of a ciphertext (and, for a bad leaf dimension, the per-leaf final rotations)
  seeded    the fused call with every a_i held as its PRG seed and regenerated on each call
  abi       the existing entry points, one call per leaf: cleanUp (copy + hb_scale_down), hb_break_into_digits, then
            hb_hoisted_linear_map (native) or hb_block_linear_map with n1 = 1 (bad dimension), accumulating
  steps     HElib's step-by-step engine path: per leaf the same cleanUp and digits, hb_automorph_keyswitch_digits per
            amount, MulAdd per diagonal, and in a bad dimension smartAutomorph of the per-leaf sum through single steps
The outer levels of rec_mul produce the leaf inputs and are the same work in every form, so the forms start from the leaf
inputs: leaf 0 over S (the unrotated path), every other leaf over S | special.  Workloads: config 5's ring (m = 21845,
p = 2) with its real dimensions 4 x 16 x bad 16 (64 leaves of the bad dimension of generator 21591), and config 3's ring
(m = 2^17, p = 257) with synthetic 16 x 16 native dimensions (16 leaves of 16 amounts), B = 1 and 8 ciphertexts.  The
four outputs are compared bit for bit.  Reports the medians with their ranges, the algorithmic GB/s of the fused call's
kernels (hb_ctx_profile), the device memory the engine holds and the card.  1 GPU; writes nothing to disk."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_block_linear_map import card, rotations  # noqa: E402
from bench_bsgs import composed  # noqa: E402

RINGS = {
    "cfg5": {"name": "m=21845 p=2 bits=580 c=2 (thin bootstrapping)", "m": 21845, "p": 2, "bits": 580, "c": 2},
    "cfg3": {"name": "bgv m=2^17 p=257 bits=1500 c=3", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3},
}
# (label, leaves = product of the outer dimensions' orders, leaf generator, leaf order D, bad leaf dimension).  Config 5's
# dimensions sorted as MatMulDimComp sorts them: orders 4 and 16 outside, the bad 16 (generator 21591) as the leaves.
WORKLOADS = {
    "cfg5": ("4x16xbad16", 64, 21591, 16, True),
    "cfg3": ("16x16", 16, 5, 16, False),
}


def leaf_amounts(m, gen, D):
    return [pow(gen, i, m) for i in range(D)], pow(gen, -D, m)


def _clean(E, x0, x1, S, ext, p, W0, W1):
    """cleanUp of one leaf of every item: a copy into W0/W1 and the mod-down to S when the leaf is over S | special."""
    if not ext:
        return x0, x1
    Sp = sorted(S + E.special)
    E.pointwise("copy", W0 + W1, x0 + x1, Sp)
    E.scale_down(W0 + W1, Sp, S, p)
    return W0, W1


def existing_abi(E, X0, X1, ext, S, ks, EA, EB, cs, A0, A1, p, cs1=None, kf=1, EAf=None, EBf=None, W0=None, W1=None, DG=None):
    """The leaves through the existing entry points, one call per leaf."""
    Sp = sorted(S + E.special)
    E.zero_rows(A0 + A1, Sp)
    for l in range(len(X0[0])):
        c0, c1 = _clean(E, [x[l] for x in X0], [x[l] for x in X1], S, ext[l], p, W0, W1)
        dg = E.break_into_digits(c1, S, DG)
        if cs1 is not None:
            E.block_linear_map(dg, S, c0, c1, ks, EA, EB, [1], [None], [None], [[c] for c in cs[l]], A0, A1,
                               consts1=[[c] for c in cs1[l]], kfinal=kf, evkf_a=EAf, evkf_b=EBf, ptxt_space=p, accumulate=True)
            continue
        live = [t for t, c in enumerate(cs[l]) if c is not None]   # hb_hoisted_linear_map takes no zero diagonal
        if live:
            E.hoisted_linear_map(dg, S, c0, c1, [ks[t] for t in live], [cs[l][t] for t in live], [EA[t] for t in live],
                                 [EB[t] for t in live], A0, A1, accumulate=True)


def step_by_step(E, X0, X1, ext, S, ks, EA, EB, cs, A0, A1, p, cs1=None, kf=1, EAf=None, EBf=None, W0=None, W1=None, DG=None,
                 R0=None, R1=None, Y0=None, Y1=None, Z0=None, Z1=None, one=None, tmp=None):
    """The leaves through single engine steps: cleanUp, digits, the hoisted rotations, MulAdd, and smartAutomorph of
    every bad leaf's second sum."""
    Sp = sorted(S + E.special)
    nit = len(X0)
    E.zero_rows(A0 + A1, Sp)
    for l in range(len(X0[0])):
        c0, c1 = _clean(E, [x[l] for x in X0], [x[l] for x in X1], S, ext[l], p, W0, W1)
        dg = E.break_into_digits(c1, S, DG)
        rotations(E, dg, S, c0, c1, ks, EA, EB, R0, R1)
        if cs1 is not None:
            E.zero_rows(Y0 + Y1, Sp)
        for t in range(len(ks)):
            r0, r1 = [r[t] for r in R0], [r[t] for r in R1]
            for c, (a0, a1) in ((cs[l][t], (A0, A1)), (cs1[l][t] if cs1 is not None else None, (Y0, Y1))):
                if c is not None:
                    E.muladd(a0, r0, [c] * nit, Sp)
                    E.muladd(a1, r1, [c] * nit, Sp)
        if cs1 is not None:
            composed(E, [[y] for y in Y0], [[y] for y in Y1], S, [kf], [[one]], [EAf], [EBf], Z0, Z1, 1, p, tmp=tmp)
            E.pointwise("add", A0 + A1, Z0 + Z1, Sp)


def run_ring(key, Bs, runs, target_s):
    import numpy as np
    import torch
    from helib_b200 import Chain, Engine
    R = RINGS[key]
    label, nl, gen, D, bad = WORKLOADS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"])
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, device=0)
    E.set_stream(torch.cuda.current_stream().cuda_stream)
    p = R["p"]
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, B = len(ch.digits), max(Bs)
    ks, kf = leaf_amounts(ch.m, gen, D)
    ext = [0] + [1] * (nl - 1)
    X0 = [[E.poly() for _ in range(nl)] for _ in range(B)]
    X1 = [[E.poly() for _ in range(nl)] for _ in range(B)]
    E.randomize([x for it in X0 + X1 for x in it], Sp, 1)
    CS = [[E.poly() for _ in ks] for _ in range(nl)]
    CS1 = [[E.poly() for _ in ks] for _ in range(nl)] if bad else None
    E.randomize([x for r in CS + (CS1 or []) for x in r], Sp, 2)

    def mats(kk, seed):
        EB = [None if k == 1 else [E.poly() for _ in range(nd)] for k in kk]
        EA = [None if k == 1 else [E.poly() for _ in range(nd)] for k in kk]
        SA = [None if k == 1 else E.seeded(nd, Sp, seed + j) for j, k in enumerate(kk)]
        for j, k in enumerate(kk):
            if k != 1:
                E.randomize(EB[j], Sp, seed + 500 + j)
                E.randomize(EA[j], Sp, seed + j)
        return EA, EB, SA
    EA, EB, SA = mats(ks, 1000)
    EAf, EBf, SAf = mats([kf], 3000) if bad else ([None], [None], [None])
    one = E.poly(np.ones((E.np, E.N), dtype=np.uint64), Sp)
    out = []
    for b in Bs:
        x0, x1 = X0[:b], X1[:b]
        outs = {f: ([E.poly() for _ in range(b)], [E.poly() for _ in range(b)]) for f in ("fused", "seeded", "abi", "steps")}
        W0, W1, Y0, Y1, Z0, Z1 = ([E.poly() for _ in range(b)] for _ in range(6))
        DG = [[E.poly() for _ in range(nd)] for _ in range(b)]
        R0 = [[E.poly() for _ in ks] for _ in range(b)]
        R1 = [[E.poly() for _ in ks] for _ in range(b)]
        tmp = [[E.poly() for _ in range(b)] for _ in range(5)]
        extra = dict(cs1=CS1, kf=kf, EAf=EAf[0], EBf=EBf[0]) if bad else {}
        fx = dict(ext=ext, consts1=CS1, kfinal=kf, evkf_b=EBf[0], ptxt_space=p) if bad else dict(ext=ext, ptxt_space=p)
        forms = {
            "fused": lambda: E.full_linear_map_leaves(x0, x1, S, ks, EA, EB, CS, *outs["fused"], evkf_a=EAf[0], **fx),
            "seeded": lambda: E.full_linear_map_leaves(x0, x1, S, ks, SA, EB, CS, *outs["seeded"], evkf_a=SAf[0], **fx),
            "abi": lambda: existing_abi(E, x0, x1, ext, S, ks, EA, EB, CS, *outs["abi"], p, W0=W0, W1=W1, DG=DG, **extra),
            "steps": lambda: step_by_step(E, x0, x1, ext, S, ks, EA, EB, CS, *outs["steps"], p, W0=W0, W1=W1, DG=DG, R0=R0,
                                          R1=R1, Y0=Y0, Y1=Y1, Z0=Z0, Z1=Z1, one=one, tmp=tmp, **extra),
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
        for kname, k in prof.items():
            kern[kname] = {"launches": k["launches"], "ms": k["ms"], "alg_GB": k["bytes"] / 1e9,
                           "alg_GB_per_s": k["bytes"] / 1e9 / (k["ms"] / 1e3) if k["ms"] else None}
        rec = {"ring": key, "ring_name": R["name"], "m": ch.m, "phim": E.N, "rows": len(Sp), "digits": nd, "dims": label,
               "leaves": nl, "amounts": len(ks), "bad": bad, "items": b, "device_GB": E.stats()["device_bytes"] / 1e9,
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
        raise SystemExit("bench_full_linear_map.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.items.split(",")], a.runs, a.window)
    print(json.dumps({"metric": "full_linear_map_leaves", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs),
                      "fused_faster_than_steps_everywhere": all(r["speedup_fused_vs_steps"] > 1 for r in recs),
                      "fused_faster_than_abi_everywhere": all(r["speedup_fused_vs_abi"] > 1 for r in recs)}))


if __name__ == "__main__":
    main()
