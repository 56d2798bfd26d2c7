#!/usr/bin/env python
"""bench_poly_eval.py -- the leaf sums of polyEval (src/polyEval.cpp:129-389): every simplePolyEval leaf of one
evaluation, sum_i s_{i,r} X^i + c_r, for B ciphertexts.

polyEval's heuristic picks k baby steps and about deg/k leaves of up to k terms.  The baby power X^i sits ceil(log2 i)
primes below x (one prime per multiplication level); a leaf's sum lives on x's prime set, so each lower power is modded up
into it.  Compares, alternating in one process on the same inputs:
  fused      one hb_ctxt_scaled_sums call for all leaves (k1_scaled_sums)
  composed   per leaf term what the transcribed loop runs: a copy of the power, hb_add_primes_and_scale into the leaf's set
             (a lower power), hb_scale_rows by the term's scalar, hb_pointwise ADD into the leaf; one ADD of the constant
on config 3's ring (BGV m = 2^17, p = 257) and config 5's (m = 21845, p = 2), degrees 16, 64 and 257, B = 1 and 8.  The
two outputs must be bit-identical.  Reports medians and ranges over --runs, the speed-up, k1_scaled_sums's ms and
algorithmic GB/s (hb_ctx_profile, a separate pass) and the card with its power limit.

--whole also times the evaluation as a whole at fixed prime sets (the "eval" records): polyEval's recursion
(PatersonStockmeyer, degPowerOfTwo, recursivePolyEval and the monic adjustment's extra term) walked on a random
polynomial, the baby and giant powers and every product through batched hb_mul_relin_moddown of copies (a product drops one
ctxt prime, down to two; HElib's polyEval multiplies distinct stored powers, so no square arises), additions as addCtxt
runs them (hb_add_primes_and_scale of the lower operand, then ADD), and all leaf sums formed before the recursion, fused or
composed as above.  Reports evaluations/s of each form and the share of its time the leaf sums take (the leaf-sum step
timed alone on the same powers).  The two forms' results must be bit-identical.  1 GPU; writes nothing to disk."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RINGS = {
    "cfg3": {"name": "bgv m=2^17 p=257 bits=1500 c=3", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3},
    "cfg5": {"name": "bgv m=21845 p=2 bits=580 c=2", "m": 21845, "p": 2, "bits": 580, "c": 2},
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


def choose_k(deg):   # polyEval's heuristic (src/polyEval.cpp:147-155)
    kk = int(math.sqrt(deg / 2.0))
    k = 1 << max(0, (kk - 1).bit_length()) if kk > 0 else 1
    if (k == 16 and deg > 167) or (k > 16 and k > 1.44 * kk):
        k //= 2
    return k


# ---- polyEval's recursion on a polynomial mod p (the mirror's hb::polyEval, include/helib_b200_ctxt.hpp)
def pdeg(a):
    return len(a) - 1


def pnorm(a):
    while a and a[-1] == 0:
        a.pop()
    return a


def pset(a, i, c=1):
    if i > pdeg(a):
        if c == 0:
            return
        a.extend([0] * (i + 1 - len(a)))
    a[i] = c
    pnorm(a)


def nextpow2(m):
    k = 0
    while (1 << k) < m:
        k += 1
    return k


def divrem_mod(r, q, p):
    dq, s = pdeg(q), [v % p for v in r]
    c = [0] * max(0, pdeg(r) - dq + 1)
    for i in range(pdeg(r), dq - 1, -1):
        t = s[i]
        c[i - dq] = t
        for j in range(dq + 1):
            s[i - dq + j] = (s[i - dq + j] - t * q[j]) % p
    return pnorm(c), pnorm(s[:max(0, min(dq, len(s)))])


class Walk:
    """The recursion's shape and its ciphertext operations on `ops`.  dry: record the simplePolyEval leaves; otherwise take
    the leaf results from `leaves`, in the same order.  A leaf result of None is an empty ciphertext."""

    def __init__(self, ops, k, p, giant_base):
        self.ops, self.k, self.p, self.dry, self.recorded, self.leaves, self.giant = ops, k, p, True, [], None, {}
        self.giant_base = giant_base

    def simple(self, poly):
        if self.dry:
            self.recorded.append(list(poly))
            return None
        return self.leaves.pop(0)

    def gpow(self, e):
        if e not in self.giant:
            self.giant[e] = self.giant_base() if e == 1 else self.ops.mul(self.gpow(e - (1 << (nextpow2(e) - 1))),
                                                                          self.gpow(1 << (nextpow2(e) - 1)))
        return self.giant[e]

    def mul(self, a, b):
        return None if self.dry or a is None or b is None else self.ops.mul(a, b)   # multiplyBy(empty) empties

    def add(self, a, b):
        if self.dry or b is None:
            return a
        return self.ops.copy(b) if a is None else self.ops.add(a, b)

    def ps(self, poly, t, delta):
        k, p = self.k, self.p
        if pdeg(poly) <= k:
            return self.simple(poly)
        r, q = pnorm(poly[:k * t]), poly[k * t:]
        pset(r, pdeg(q), (r[pdeg(q)] if pdeg(q) < len(r) else 0) - 1)
        c, s = divrem_mod(r, q, p)
        pset(s, pdeg(q))
        ret = self.ps(q, t // 2, delta)
        tmp = self.simple(c)
        tmp = self.add(tmp, None if self.dry else self.gpow(t))
        ret = self.mul(ret, tmp)
        return self.add(ret, self.ps(s, t // 2, delta))

    def deg_pow2(self, poly):
        k = self.k
        if pdeg(poly) <= k:
            return self.simple(poly)
        n = 1 << nextpow2(pdeg(poly) // k)
        r, q = pnorm(poly[:(n - 1) * k]), list(poly[(n - 1) * k:])
        pset(r, (n - 1) * k)
        q = [-1] if not q else pnorm([q[0] - 1] + q[1:])
        ret = self.ps(r, n // 2, 0)
        tmp = self.simple(q)
        i = 1
        while i < n and not self.dry:
            tmp = self.mul(tmp, self.gpow(i))
            i *= 2
        return self.add(ret, tmp)

    def recursive(self, poly):
        k = self.k
        if pdeg(poly) <= k:
            return self.simple(poly)
        delta, n = pdeg(poly) % k, -(-pdeg(poly) // k)
        t = 1 << nextpow2(n)
        if n == t:
            return self.deg_pow2(poly)
        if n == t - 1 and delta == 0:
            return self.ps(poly, t // 2, delta)
        t //= 2
        u = pdeg(poly) - k * (t - 1)
        r, q = pnorm(poly[:u]), list(poly[u:])
        q = [-1] if not q else pnorm([q[0] - 1] + q[1:])
        pset(r, u)
        ret = self.ps(q, t // 2, 0)
        if not self.dry:
            tmp = self.gpow(u // k)
            if delta:
                tmp = self.ops.mul(tmp, self.ops.baby(delta))
            ret = self.mul(ret, tmp)
        return self.add(ret, self.recursive(r))


class Ops:
    """Batched ciphertexts (B items of two parts) at fixed prime sets S[:L], on a pool of polys reused between
    evaluations (freeing a poly synchronises the stream)."""

    def __init__(self, E, S, p, EA, EB, b):
        self.E, self.S, self.p, self.EA, self.EB, self.b = E, S, p, EA, EB, b
        self.pool, self.used, self.powers = [], 0, {}

    def fresh(self, L):
        while self.used + 2 * self.b > len(self.pool):
            self.pool.append(self.E.poly())
        ps = self.pool[self.used:self.used + 2 * self.b]
        self.used += 2 * self.b
        return (ps[:self.b], ps[self.b:], L)

    def copy(self, a):
        c = self.fresh(a[2])
        for k in range(2):
            self.E.pointwise("copy", c[k], a[k], self.S[:a[2]])
        return c

    def mul(self, a, b):
        A, B = self.copy(a), self.copy(b)
        L = min(a[2], b[2])
        for X in (A, B):
            if X[2] > L:
                self.E.scale_down(X[0] + X[1], self.S[:X[2]], self.S[:L], self.p)
        Lo = max(L - 1, 2)
        self.E.mul_relin_moddown(A[0], A[1], B[0], B[1], self.S[:L], self.S[:Lo], self.p, self.EA, self.EB)
        return (A[0], A[1], Lo)

    def add(self, a, b):   # addCtxt: the lower operand is modded up to the higher one's set
        if a[2] < b[2]:
            self.E.add_primes_and_scale(a[0] + a[1], self.S[:a[2]], self.S[a[2]:b[2]])
            a = (a[0], a[1], b[2])
        elif b[2] < a[2]:
            b = self.copy(b)
            self.E.add_primes_and_scale(b[0] + b[1], self.S[:b[2]], self.S[b[2]:a[2]])
        for k in range(2):
            self.E.pointwise("add", a[k], b[k], self.S[:a[2]])
        return a

    def baby(self, e):
        if e not in self.powers:
            h = 1 << (nextpow2(e) - 1)
            self.powers[e] = self.mul(self.baby(e - h), self.baby(h))
        return self.powers[e]


def leaf_tables(ch, S, leaves, levels, rng):
    """Per leaf j and term i: random nonzero residues on the rows of X^i's set (zero on the rest), a random constant on
    the leaf's set (the highest of its terms' sets), and the composed form's scalars (s times the mod-up factor's inverse)."""
    nin = max(pdeg(l) for l in leaves)
    nU = max(levels[i] for i in range(1, nin + 1))
    scal = np.zeros((len(leaves), nin, nU), dtype=np.uint64)
    comp = np.zeros_like(scal)
    cst = np.zeros((len(leaves), nU), dtype=np.uint64)
    lvl = []
    for j, l in enumerate(leaves):
        top = max(levels[i] for i in range(1, pdeg(l) + 1))
        lvl.append(top)
        for r in range(top):
            cst[j, r] = int(rng.integers(0, ch.primes[S[r]]))
        for i in range(1, pdeg(l) + 1):
            P = 1
            for row in S[levels[i]:top]:
                P *= ch.primes[row]
            for r in range(levels[i]):
                q = ch.primes[S[r]]
                v = int(rng.integers(1, q))
                scal[j, i - 1, r] = v
                comp[j, i - 1, r] = v * pow(P % q, -1, q) % q
    return scal, comp, cst, lvl


def run_eval(key, degs, Bs, runs):
    """Whole evaluations at fixed prime sets, fused against composed leaf sums."""
    import torch
    from helib_b200 import Chain
    from helib_b200.engine import Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"], lib=None)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special)
    S, p = ch.ctxt, R["p"]
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    EA, EB = [E.poly() for _ in range(nd)], [E.poly() for _ in range(nd)]
    E.randomize(EA, full, 11)
    E.randomize(EB, full, 12)
    out = []
    for deg in degs:
        rng = np.random.default_rng(deg)
        poly = [int(v) for v in rng.integers(0, p, size=deg + 1)]
        poly[-1] = 1 + int(rng.integers(0, p - 1))
        k = choose_k(deg)
        n = -(-deg // k)
        pow2 = n == 1 << nextpow2(n)
        extra = 0
        if not pow2:   # the monic adjustment (src/polyEval.cpp:178-219)
            top = poly[-1]
            if n * k != deg or math.gcd(top, p) != 1:
                extra = (1 - (poly[n * k] if n * k <= deg else 0)) % p
                pset(poly, n * k)
            elif top != 1:
                inv = pow(top, -1, p)
                poly = pnorm([v * inv % p for v in poly])
        for b in Bs:
            ops = Ops(E, S, p, EA, EB, b)
            x = ops.fresh(len(S))
            E.randomize(x[0] + x[1], S, 77)
            walk = Walk(ops, k, p, lambda: ops.baby(k))
            (walk.deg_pow2 if pow2 else walk.recursive)(poly)   # dry: the leaves
            leaves = walk.recorded
            base = ops.used

            def powers():
                ops.used, ops.powers, walk.giant = base, {1: x}, {}
                for i in range(1, max(max(pdeg(l) for l in leaves), 1) + 1):
                    ops.baby(i)

            powers()
            levels = {i: ops.powers[i][2] for i in ops.powers}
            scal, comp, cst, lvl = leaf_tables(ch, S, [l for l in leaves if pdeg(l) >= 1], levels, rng)
            nU = scal.shape[2]

            def sums(fused):
                live = [l for l in leaves if pdeg(l) >= 1]
                outs = [ops.fresh(lv) for lv in lvl]
                nin = scal.shape[1]
                X = [ops.powers[i] for i in range(1, nin + 1)]
                if fused:
                    E.ctxt_scaled_sums([[X[i][0][t] for i in range(nin)] for t in range(b)],
                                       [[X[i][1][t] for i in range(nin)] for t in range(b)],
                                       [[o[0][t] for o in outs] for t in range(b)], [[o[1][t] for o in outs] for t in range(b)],
                                       S[:nU], scal, cst)
                else:
                    tmp = ops.fresh(len(S))
                    for j, (l, o) in enumerate(zip(live, outs)):
                        for i in range(1, pdeg(l) + 1):
                            Xi = X[i - 1]
                            for part in range(2):
                                E.pointwise("copy", tmp[part], Xi[part], S[:Xi[2]])
                            if Xi[2] < o[2]:
                                E.add_primes_and_scale(tmp[0] + tmp[1], S[:Xi[2]], S[Xi[2]:o[2]])
                            E.scale_rows(tmp[0] + tmp[1], S[:o[2]], comp[j, i - 1, :o[2]])
                            for part in range(2):
                                E.pointwise("copy" if i == 1 else "add", o[part], tmp[part], S[:o[2]])
                        for t in range(b):   # the constant: cst[j, r] on every coefficient of row r
                            E.pointwise("add", [o[0][t]], [cconst[j]], S[:o[2]])
                res, it = [], iter(outs)
                for l in leaves:
                    res.append(next(it) if pdeg(l) >= 1 else None)
                return res

            cconst = []
            for j in range(len(lvl)):
                cp = E.poly()
                d = np.zeros((len(ch.primes), E.N), dtype=np.uint64)
                for r in range(lvl[j]):
                    d[S[r]] = cst[j, r]
                cp.upload(d, S[:lvl[j]])
                cconst.append(cp)

            def evaluation(fused):
                powers()
                walk.dry, walk.leaves = False, sums(fused)
                ret = (walk.deg_pow2 if pow2 else walk.recursive)(poly)
                if extra:
                    top_term = ops.copy(walk.gpow(n))
                    sc = np.array([(p - extra) % ch.primes[S[r]] for r in range(top_term[2])], dtype=np.uint64)
                    E.scale_rows(top_term[0] + top_term[1], S[:top_term[2]], sc)
                    ret = ops.add(ret, top_term)
                walk.dry = True
                return ret

            def sums_only(fused):
                ops.used = mark
                sums(fused)

            def timed(fn, *a):
                torch.cuda.synchronize()
                E.mark_begin()
                r = fn(*a)
                return E.mark_end(), r

            for f in (True, False):   # warm every shape
                timed(evaluation, f)
            powers()
            mark = ops.used
            for f in (True, False):
                timed(sums_only, f)
            ms = {"fused": [], "composed": []}
            sms = {"fused": [], "composed": []}
            for _ in range(runs):
                for f, name in ((True, "fused"), (False, "composed")):
                    ms[name].append(timed(evaluation, f)[0])
                powers()
                mark = ops.used
                for f, name in ((True, "fused"), (False, "composed")):
                    sms[name].append(timed(sums_only, f)[0])
            got = {}
            for f, name in ((True, "fused"), (False, "composed")):
                r = evaluation(f)
                got[name] = [r[part][t].download(S[:r[2]])[S[:r[2]]] for part in range(2) for t in range(b)]
            identical = all(np.array_equal(u, v) for u, v in zip(got["fused"], got["composed"]))
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            smed = {f: sorted(v)[len(v) // 2] for f, v in sms.items()}
            rec = {"ring": key, "ring_name": R["name"], "kind": "eval", "phim": E.N, "ctxt_primes": len(S), "degree": deg,
                   "k": k, "leaves": len(leaves), "items": b,
                   "median_ms": {f: round(v, 3) for f, v in med.items()},
                   "range_ms": {f: [round(min(v), 3), round(max(v), 3)] for f, v in ms.items()},
                   "evals_per_s": {f: b / (v / 1e3) for f, v in med.items()},
                   "sums_median_ms": {f: round(v, 3) for f, v in smed.items()},
                   "sums_share": {f: smed[f] / med[f] for f in med},
                   "speedup_fused_vs_composed": med["composed"] / med["fused"],
                   "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
            del ops, x, walk, cconst
    del EA, EB
    E.close()
    return out


def run_ring(key, degs, Bs, runs):
    import torch
    from helib_b200 import Chain
    from helib_b200.engine import Engine
    R = RINGS[key]
    ch = Chain(R["m"], R["p"], 1, R["bits"], R["c"], lib=None)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special)
    S = ch.ctxt
    qS = np.array([ch.primes[r] for r in S], dtype=object)
    rng = np.random.default_rng(5)
    out = []
    for deg in degs:
        k = choose_k(deg)
        nleaf = -(-(deg + 1) // (k + 1))
        sets = [S[:len(S) - (i - 1).bit_length()] for i in range(1, k + 1)]   # X^i: ceil(log2 i) primes lower
        scal = np.zeros((nleaf, k, len(S)), dtype=np.uint64)
        for j in range(nleaf):
            for i in range(k):
                for r in range(len(sets[i])):
                    scal[j, i, r] = int(rng.integers(1, ch.primes[S[r]]))
        cst = np.stack([np.array([int(rng.integers(0, q)) for q in qS], dtype=np.uint64) for _ in range(nleaf)])
        for b in Bs:
            Xs = [[[E.poly() for _ in range(k)] for _ in range(b)] for _ in range(2)]
            for t in range(b):
                for i in range(k):
                    E.randomize([Xs[0][t][i], Xs[1][t][i]], sets[i], 100 * t + i)
            F = [[[E.poly() for _ in range(nleaf)] for _ in range(b)] for _ in range(2)]
            C = [[[E.poly() for _ in range(nleaf)] for _ in range(b)] for _ in range(2)]
            tmp = [E.poly() for _ in range(2)]
            cpoly = [E.poly() for _ in range(nleaf)]
            for j in range(nleaf):   # the constant as a poly: cst[j, r] on every coefficient of row r
                d = np.zeros((len(ch.primes), E.N), dtype=np.uint64)
                for r, row in enumerate(S):
                    d[row] = cst[j, r]
                cpoly[j].upload(d, S)
            # composed: rows *= P mod q on a mod-up, so the scaled step takes s * P^-1 there (the same result)
            sc_comp = np.zeros_like(scal)
            for i in range(k):
                P = 1
                for row in S[len(sets[i]):]:
                    P *= ch.primes[row]
                for r in range(len(sets[i])):
                    q = ch.primes[S[r]]
                    sc_comp[:, i, r] = [int(v) * pow(P % q, -1, q) % q for v in scal[:, i, r]]

            def fused():
                E.ctxt_scaled_sums(Xs[0], Xs[1], F[0], F[1], S, scal, cst)

            def composed():
                for t in range(b):
                    for j in range(nleaf):
                        first = True
                        for i in range(k):
                            for part in range(2):
                                E.pointwise("copy", [tmp[part]], [Xs[part][t][i]], sets[i])
                            if len(sets[i]) < len(S):
                                E.add_primes_and_scale(tmp, sets[i], S[len(sets[i]):])
                            E.scale_rows(tmp, S, sc_comp[j, i])
                            for part in range(2):
                                E.pointwise("copy" if first else "add", [C[part][t][j]], [tmp[part]], S)
                            first = False
                        E.pointwise("add", [C[0][t][j]], [cpoly[j]], S)

            forms = {"fused": fused, "composed": composed}

            def timed(fn):
                torch.cuda.synchronize()
                E.mark_begin()
                fn()
                return E.mark_end()

            for fn in forms.values():
                timed(fn)
            ms = {f: [] for f in forms}
            for _ in range(runs):
                for f, fn in forms.items():
                    ms[f].append(timed(fn))
            fused()
            composed()
            identical = all(np.array_equal(F[p][t][j].download(S)[S], C[p][t][j].download(S)[S])
                            for p in range(2) for t in range(b) for j in range(nleaf))
            torch.cuda.synchronize()
            E.profile(True)
            fused()
            prof = {r["kernel"]: r for r in E.profile_results()}
            E.profile(False)
            kp = prof.get("k1_scaled_sums", {"ms": 0.0, "bytes": 0, "launches": 0})
            med = {f: sorted(v)[len(v) // 2] for f, v in ms.items()}
            rec = {"ring": key, "ring_name": R["name"], "phim": E.N, "ctxt_primes": len(S), "degree": deg, "k": k,
                   "leaves": nleaf, "items": b,
                   "median_ms": {f: round(v, 4) for f, v in med.items()},
                   "range_ms": {f: [round(min(v), 4), round(max(v), 4)] for f, v in ms.items()},
                   "speedup_fused_vs_composed": med["composed"] / med["fused"],
                   "k1_scaled_sums": {"launches": kp["launches"], "ms": kp["ms"], "alg_GB": kp["bytes"] / 1e9,
                                      "alg_GB_per_s": kp["bytes"] / 1e9 / (kp["ms"] / 1e3) if kp["ms"] else None},
                   "bit_identical": identical}
            print(json.dumps(rec), flush=True)
            out.append(rec)
            del Xs, F, C, tmp, cpoly
    E.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", default="cfg3,cfg5")
    ap.add_argument("--degrees", default="16,64,257")
    ap.add_argument("--items", default="1,8")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--whole", action="store_true", help="also time whole evaluations (the eval records)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_poly_eval.py needs a CUDA device")
    name, pl = card()
    recs = []
    for key in a.rings.split(","):
        recs += run_ring(key, [int(x) for x in a.degrees.split(",")], [int(x) for x in a.items.split(",")], a.runs)
        if a.whole:
            recs += run_eval(key, [int(x) for x in a.degrees.split(",")], [int(x) for x in a.items.split(",")], a.runs)
    print(json.dumps({"metric": "poly_eval_leaf_sums", "card": name, "power_limit": pl, "runs_per_form": a.runs,
                      "all_bit_identical": all(r["bit_identical"] for r in recs)}))


if __name__ == "__main__":
    main()
