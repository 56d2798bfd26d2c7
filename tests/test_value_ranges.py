"""Worst-case operands at the largest admissible primes.

The kernels sum many 64x64-bit products in 128 bits and reduce once, and the register kernels keep lazy values whose
bounds ("q < 2^60", "x < 8q + 2^32", "13q + 2^49 < 2^64") hold only up to their limits.  Random residues keep a
128-bit sum near a quarter of its worst case, so a limit set a few times too high still passes every random-data test.
Here every chain is made of the largest primes below 2^60 and every value that enters a sum or a lazy network sits at
the top of its range: rows of q-1, rows alternating 0 and q-1 (in evaluation and in coefficient form), digits whose
every residue is q-1 (the constant c = -(1 + Q_0 + Q_0 Q_1 + ...), whose balanced mixed-radix digits are all -1 and
which every automorphism fixes), reduced intermediates equal to q-1, and keys, constants and accumulators at q-1.  Each
path runs at its per-launch maximum, the launch profile shows the intended kernel ran, and the result must equal the
oracle's step-by-step computation (which reduces every product on its own) bit for bit.  Every body runs on the CPU
simulator build and, marked gpu, on the H100.
"""
import math

import numpy as np
import pytest

import orc
import pyoracle as po
from helib_b200.engine import Engine
from test_bsgs import GenOps, PowOps, _reference as bsgs_reference
from test_engine_parity import oracle_mul_relin_moddown
from test_linear_map import GenOracle, _reference as linmap_reference

TOP = 1 << 60
FLOOR = TOP - (1 << 40)


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


# ---- 1. chains of the largest admissible primes

def transform_divisor(m):
    """What q - 1 must be divisible by: m for power-of-two m; for general m the order e of the roots and the Bluestein
    length L (gen_init, hb_engine.cu:1442)."""
    if m & (m - 1) == 0:
        return m
    e = 2 * m if m % 2 == 0 else m
    L = 1
    while L < 2 * m - 1:
        L *= 2
    return math.lcm(e, L)


_PRIMES = {}


def largest_primes(form, count, m):
    """The largest primes in (2^60 - 2^40, 2^60) with transform_divisor(m) | q - 1, in one of the two modulus views of
    the register kernels (Hb1Mod, hb_device_v1.cuh:69-75):
      'sp'  q = t*2^s + 1 with t odd, t < 2^32 and s >= 32 (qt != 0); taken round-robin over s = 32, 33, ... so that
            primes with s > 32 (qsh != 0) are among them;
      'gen' 2^32 does not divide q - 1 (qt = 0)."""
    key = (form, count, m)
    if key in _PRIMES:
        return _PRIMES[key]
    div = transform_divisor(m)
    out = []
    if form == "sp":
        assert div & (div - 1) == 0 and div <= 1 << 32
        per_s = []
        for s in range(32, 48):
            t, lst = (TOP - 1) >> s, []
            t -= 1 - (t & 1)
            while (t << s) + 1 > FLOOR:
                if po.is_prime((t << s) + 1):
                    lst.append((t << s) + 1)
                t -= 2
            per_s.append(lst)
        while len(out) < count:
            row = [lst.pop(0) for lst in per_s if lst]
            assert row, "not enough shift-form primes in (2^60 - 2^40, 2^60)"
            out += row
        out = out[:count]
    else:
        k = (TOP - 2) // div
        while len(out) < count:
            q = k * div + 1
            assert q > FLOOR
            if (q - 1) % (1 << 32) != 0 and po.is_prime(q):
                out.append(q)
            k -= 1
    assert all(FLOOR < q < TOP for q in out) and len(set(out)) == count
    _PRIMES[key] = out
    return out


def top_chain(lib, m, p, form, digit_sizes, nspecial, nthreads=8):
    """A po.Chain of the largest primes: ctxt primes in digits of digit_sizes primes each, then nspecial special primes;
    the engine on it and the step-by-step reference (the C++ oracle for power-of-two m, big-integer Python otherwise)."""
    nctxt = sum(digit_sizes)
    primes = largest_primes(form, nctxt + nspecial, m)
    digits, i = [], 0
    for n in digit_sizes:
        digits.append(list(range(i, i + n)))
        i += n
    ch = po.Chain(m=m, p=p, r=1, phim=po.euler_phi(m), primes=primes, ctxt=list(range(nctxt)),
                  special=list(range(nctxt, nctxt + nspecial)), digits=digits)
    if m & (m - 1) == 0:
        psis = [po.find_psi(q, m) for q in primes]
        O = orc.Oracle(ch.phim, m, primes, psis, digits, ch.special, nthreads=nthreads)
        E = Engine(m, primes, psis, digits, ch.special, lib=lib)
    else:
        O = None
        E = Engine(m, primes, None, digits, ch.special, lib=lib)
    return ch, O, E


def ptxt(ch):
    return 1 if ch.p == -1 else ch.p ** ch.r


# ---- 2. worst-case operands

def dense(ch):
    return np.zeros((len(ch.primes), ch.phim), dtype=np.uint64)


def const_rows(ch, idx, v):
    """The constant polynomial v (a Python int) on the rows idx: every evaluation of a constant is the constant, so
    every residue of row i is v mod q_i, in evaluation and in coefficient form alike."""
    out = dense(ch)
    for i in idx:
        out[i] = v % ch.primes[i]
    return out


def top(ch, idx):
    return const_rows(ch, idx, -1)


def alternating(ch, idx, phase=0):
    out = dense(ch)
    for i in idx:
        out[i][phase::2] = ch.primes[i] - 1
    return out


def to_eval(ch, O, x, idx):
    """Coefficient rows -> evaluation rows, by the oracle."""
    x = x.copy()
    if O is not None:
        O.ntt_fwd_rows(x, idx)
    else:
        roots = [po.cmod_root(q, ch.m) for q in ch.primes]
        for i in idx:
            x[i] = np.array(po.gen_fft([int(v) for v in x[i]], ch.primes[i], ch.m, roots[i]), dtype=np.uint64)
    return x


def operand(ch, O, idx, kind):
    """'top' / 'alt': rows of q-1 / of alternating 0 and q-1 in evaluation form; 'ctop' / 'calt': the same in
    coefficient form, transformed; 'cmid': coefficient rows cycling through 0, 1, q-1, the halves around q/2 and 2, q-2."""
    if kind == "top":
        return top(ch, idx)
    if kind == "alt":
        return alternating(ch, idx)
    if kind == "ctop":
        return to_eval(ch, O, top(ch, idx), idx)
    if kind == "calt":
        return to_eval(ch, O, alternating(ch, idx, 1), idx)
    assert kind == "cmid"
    x = dense(ch)
    for i in idx:
        q = ch.primes[i]
        pat = np.array([0, 1, q - 1, (q - 1) // 2, (q + 1) // 2, q // 2 - 1, 2, q - 2], dtype=np.uint64)
        x[i] = np.resize(pat, ch.phim)
    return to_eval(ch, O, x, idx)


def all_minus_one_digits(ch, S):
    """c = -(1 + Q_0 + Q_0 Q_1 + ...) over the digits of S: its balanced mixed-radix digits are all -1."""
    c, Qp = 0, 1
    for d in ch.digits:
        part = [i for i in d if i in S]
        if part:
            c -= Qp
            Qp *= ch.product(part)
    return c


def ndigits(ch, S):
    return sum(1 for d in ch.digits if any(i in S for i in d))


def kernels(E):
    return {r["kernel"] for r in E.profile_results()}


def equal(P, ref, idx):
    return bool((P.download(idx)[idx] == ref[idx]).all())


def top_keys(ch, E, n=None):
    """One key-switching matrix whose every row is q-1 (as arrays and as Polys over S | special)."""
    full = ch.ctxt + ch.special
    n = len(ch.digits) if n is None else n
    ea = np.stack([top(ch, full) for _ in range(n)])
    return ea, [E.poly(ea[i], full) for i in range(n)]


# ---- 3. paths at their per-launch maximum

R17 = 1 << 17


@pytest.mark.parametrize("case", [
    ("sp", 257, 1, "default"), ("sp", 2, 1, "default"), ("gen", -1, 1, "default"), ("sp", -1, 2, "default"),
    ("sp", 257, 2, "default"), ("sp", 257, 0, "default"), ("sp", -1, 0, "default"),
    ("sp", 257, 1, "blk_v2"), ("sp", 2, 1, "no_special"),
], ids=lambda c: "-".join(str(x) for x in c))
def test_mul_relin_moddown_register_kernels(lib, monkeypatch, case):
    """hb_mul_relin_moddown at N = 2^16 with operands at the top of their ranges, BGV p = 257, p = 2 (the mod-down's tie
    rule) and CKKS, dropping 1, 2 or no primes.  Bounds: the subscale epilogue's (old - x + 12q) * P^-1 with x < 8q + 2^32,
    old < 4q (hb_device_v1.cuh:333 in k1_fwd_blk, :431 in k1_fwd_blk_tensor); "everything stays below 13q + 2^49 < 2^64"
    (:53); k1_tensor's a0*b1 + a1*b0 in 128 bits (:882); k1_conv's target sums.  HB_BLK_V2=1 runs the TMA k2_* blk kernels,
    HB_NO_SPECIAL=1 the generic modulus view on shift-form primes."""
    form, p, ndrop, env = case
    if env == "blk_v2":
        monkeypatch.setenv("HB_BLK_V2", "1")
    if env == "no_special":
        monkeypatch.setenv("HB_NO_SPECIAL", "1")
    ch, O, E = top_chain(lib, R17, p, form, [1, 1, 2], 2)
    S_in = ch.ctxt
    S = S_in[:len(S_in) - ndrop]
    ea, EA = top_keys(ch, E)
    eb, EB = ea, EA
    kinds = [("top", "calt", "ctop", "alt"), ("cmid", "top", "alt", "ctop")]
    ops = [[operand(ch, O, S_in, k) for k in ks] for ks in kinds]
    A0, A1, B0, B1 = ([E.poly(o[k], S_in) for o in ops] for k in range(4))
    E.profile(True)
    E.mul_relin_moddown(A0, A1, B0, B1, S_in, S, ptxt(ch), EA, EB)
    E.profile(False)
    for it, o in enumerate(ops):
        r0, r1 = oracle_mul_relin_moddown(O, ch, *o, S_in, S, ptxt(ch), ea, eb)
        assert equal(A0[it], r0, S) and equal(A1[it], r1, S), it
    ran = kernels(E)
    if ndrop == 0:
        assert "k1_tensor" in ran and "k1_fwd_blk_tensor" not in ran, ran
    else:
        assert "k1_fwd_blk_tensor" in ran and "k1_tensor" not in ran, ran
        assert ("k1_conv1" if ndrop == 1 and p == -1 else "k1_conv") in ran, ran
    if env == "blk_v2":
        assert "k2_fwd_blk_subscale" in ran and not any(k.startswith(("k1_fwd_blk_sub", "k1_fwd_blk_dig")) for k in ran), ran
    assert "k1_ks_inner" in ran, ran


@pytest.mark.parametrize("p", [257, 2, -1])
@pytest.mark.parametrize("m", [64, 4096])
def test_mul_relin_moddown_generic_kernels(lib, m, p):
    """Below the register kernels: m = 64 (N = 32) takes the tensor product in k_pw_tensor, m = 4096 (N = 2048) in
    k1_tensor after the generic rescale (k_fwd_blk_subscale); operands at the top of their ranges, keys of q-1, 4 digits.
    Bounds: the 128-bit a0*b1 + a1*b0 of k_pw_tensor (hb_device.cuh, k_pointwise TENSOR) and k1_tensor
    (hb_device_v1.cuh:882), the generic transform's lazy ranges."""
    ch, O, E = top_chain(lib, m, p, "gen", [1, 1, 1, 1], 2)
    S_in, S = ch.ctxt, ch.ctxt[:-1]
    ea, EA = top_keys(ch, E)
    ops = [[operand(ch, O, S_in, k) for k in ks] for ks in [("top", "calt", "ctop", "alt"), ("cmid", "top", "top", "ctop")]]
    A0, A1, B0, B1 = ([E.poly(o[k], S_in) for o in ops] for k in range(4))
    E.profile(True)
    E.mul_relin_moddown(A0, A1, B0, B1, S_in, S, ptxt(ch), EA, EA)
    E.profile(False)
    for it, o in enumerate(ops):
        r0, r1 = oracle_mul_relin_moddown(O, ch, *o, S_in, S, ptxt(ch), ea, ea)
        assert equal(A0[it], r0, S) and equal(A1[it], r1, S), it
    ran = kernels(E)
    assert ({"k_pw_tensor"} if m == 64 else {"k1_tensor", "k_fwd_blk_subscale"}) <= ran, ran


@pytest.mark.parametrize("case", [("sp", "default"), ("gen", "default"), ("sp", "blk_v2"), ("sp", "no_special")],
                         ids=lambda c: "-".join(c))
def test_fused_relinearize_with_all_minus_one_digits(lib, monkeypatch, case):
    """hb_relinearize on the register kernels with four digits (the most the fused path takes at N = 2^16): c2 is the
    constant whose digits are all -1, so the lazy digits the digit epilogue leaves (epi 3, hb_device_v1.cuh:307-336) and
    k1_ks_inner reads are q-1 in every row; keys, c0 and c1 are q-1.  Bounds: the digit epilogue's (old - x + 12q) * Q^-1
    (:333), k1_ks_inner's HB_MAXDIG + 1 products in 128 bits (:853-856)."""
    form, env = case
    if env == "blk_v2":
        monkeypatch.setenv("HB_BLK_V2", "1")
    if env == "no_special":
        monkeypatch.setenv("HB_NO_SPECIAL", "1")
    ch, O, E = top_chain(lib, R17, 257, form, [1, 1, 1, 1], 2)
    ea, EA = top_keys(ch, E)
    for S in (ch.ctxt, ch.ctxt[:-1]):
        Sp = sorted(S + ch.special)
        c = all_minus_one_digits(ch, S)
        digs = O.break_into_digits(const_rows(ch, S, c), S)
        assert all((digs[d][i] == ch.primes[i] - 1).all() for d in range(ndigits(ch, S)) for i in Sp)
        cs = [[top(ch, S), alternating(ch, S), const_rows(ch, S, c)], [operand(ch, O, S, "ctop"), top(ch, S), const_rows(ch, S, c)]]
        C0, C1, C2 = ([E.poly(x[k], S) for x in cs] for k in range(3))
        E.profile(True)
        E.relinearize(C0, C1, C2, S, EA, EA)
        E.profile(False)
        ran = kernels(E)
        assert "k1_ks_inner" in ran and ("k2_fwd_blk_digits" if env == "blk_v2" else "k1_fwd_blk_digits") in ran, ran
        E.scale_down(C0 + C1, Sp, S, 257)
        for it, x in enumerate(cs):
            r0, r1 = O.relinearize(x[0], x[1], x[2], S, ea, ea)
            O.scale_down(r0, Sp, S, 257); O.scale_down(r1, Sp, S, 257)
            assert equal(C0[it], r0, S) and equal(C1[it], r1, S), (len(S), it)


def small_chain(lib, m=64, p=257, nd=8, per=1, nspecial=2):
    return top_chain(lib, m, p, "gen", [per] * nd, nspecial)


@pytest.mark.parametrize("m", [64, 4096])
def test_keyswitch_entry_points_with_the_most_digits(lib, m):
    """hb_keyswitch_digits, hb_keyswitch_digits_fused and hb_automorph_keyswitch_digits with HB_MAXDIG = 8 digits of q-1,
    keys of q-1 and c0, c1 of q-1.  Bound: k_ks_inner's at most HB_MAXDIG + 1 products below 2^120 in 128 bits
    (hb_device.cuh:715-726)."""
    ch, O, E = small_chain(lib, m)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    assert nd == 8
    ea, EA = top_keys(ch, E)
    digs = np.stack([top(ch, Sp) for _ in range(nd)])
    D = [[E.poly(digs[i], Sp) for i in range(nd)]]
    # plain inner product, added to outputs that hold q-1
    O0, O1 = E.poly(top(ch, Sp), Sp), E.poly(top(ch, Sp), Sp)
    E.profile(True)
    E.keyswitch_digits(D, Sp, EA, EA, [O0], [O1])
    r0, r1 = top(ch, Sp), top(ch, Sp)
    O.keyswitch_digits(digs, Sp, ea, ea, r0, r1)
    assert equal(O0, r0, Sp) and equal(O1, r1, Sp)
    # fused: addPrimesAndScale of c0, c1 folded in
    P = ch.product(ch.special)
    scal = [P % ch.primes[r] if r in S else 0 for r in Sp]
    C0, C1 = E.poly(top(ch, Sp), Sp), E.poly(alternating(ch, Sp), Sp)
    E.keyswitch_digits_fused(D, Sp, EA, EA, [C0], [C1], scal)
    r0, r1 = top(ch, S), alternating(ch, S)
    O.add_primes_and_scale(r0, S, ch.special); O.add_primes_and_scale(r1, S, ch.special)
    O.keyswitch_digits(digs, Sp, ea, ea, r0, r1)
    assert equal(C0, r0, Sp) and equal(C1, r1, Sp)
    # hoisted automorphism
    c0 = top(ch, S)
    for k in (3, m - 1):
        Q0, Q1 = E.poly(), E.poly()
        E.automorph_keyswitch_digits(D, S, [E.poly(c0, S)], k, EA, EA, [Q0], [Q1])
        r0 = c0.copy(); O.automorph(r0, S, k); O.add_primes_and_scale(r0, S, ch.special)
        r1 = O.zeros()
        O.keyswitch_digits(digs, Sp, ea, ea, r0, r1)     # the digits are constants: automorph leaves them
        assert equal(Q0, r0, Sp) and equal(Q1, r1, Sp), k
    E.profile(False)
    assert "k_ks_inner" in kernels(E), kernels(E)


@pytest.mark.parametrize("m", [64, 4096])
def test_muladd_and_tensor_with_q_minus_one(lib, m):
    """hb_muladd (dst + a*b) and hb_tensor (a0*b1 + a1*b0 in 128 bits) with every input q-1 and alternating rows."""
    ch, O, E = small_chain(lib, m, nd=2)
    S = sorted(ch.ctxt + ch.special)
    for a, b in ((top(ch, S), top(ch, S)), (alternating(ch, S), top(ch, S))):
        D = E.poly(top(ch, S), S)
        E.muladd([D], [E.poly(a, S)], [E.poly(b, S)], S)
        ref = a.copy(); O.pointwise("mul", ref, b, S)
        acc = top(ch, S); O.pointwise("add", acc, ref, S)
        assert equal(D, acc, S)
    x = [top(ch, S), operand(ch, O, S, "ctop"), top(ch, S), alternating(ch, S)]
    X = [E.poly(v, S) for v in x]
    Y = [E.poly() for _ in range(3)]
    E.tensor([X[0]], [X[1]], [X[2]], [X[3]], [Y[0]], [Y[1]], [Y[2]], S)
    for Yk, rk in zip(Y, O.tensor(*x, S)):
        assert equal(Yk, rk, S)


def test_tensor_register_kernel_with_q_minus_one(lib):
    """k1_tensor at N = 2^16: a0*b1 + a1*b0 summed in 128 bits (hb_device_v1.cuh:882), inputs q-1."""
    ch, O, E = top_chain(lib, R17, 257, "sp", [1, 1], 1)
    S = ch.ctxt
    x = [top(ch, S), top(ch, S), top(ch, S), alternating(ch, S)]
    X = [E.poly(v, S) for v in x]
    E.profile(True)
    E.tensor([X[0]], [X[1]], [X[2]], [X[3]], [X[0]], [X[1]], [X[2]], S)
    E.profile(False)
    for Xk, rk in zip(X, O.tensor(*x, S)):
        assert equal(Xk, rk, S)
    assert "k1_tensor" in kernels(E), kernels(E)


def test_conversions_from_many_primes_with_coefficient_extremes(lib):
    """addPrimes, scaleDownToSet (p = 1, 2, 257; the special primes dropped, and two ctxt primes with them) and
    breakIntoDigits from 16 source primes at the top of the 60-bit range, with coefficients placed at the extremes of the
    balanced range: 0, +-1, Q/2 and its neighbours, and -1 mod Q.  Bound: the conversion's 128-bit sums over at most HB_MAXROWS source primes
    (hb_device.cuh:568-572)."""
    ch, O, E = small_chain(lib, 4096, nd=8, per=2, nspecial=3)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    Q = ch.product(S)
    pat = [0, 1, Q - 1, Q // 2, Q // 2 + 1, (Q - 1) // 2, Q - 2, Q // 2 - 1, 2, Q // 3]
    vals = [pat[j % len(pat)] for j in range(ch.phim)]
    x = O.zeros()
    O.fft_bigpoly(orc.ints_to_limbs(vals, (Q.bit_length() + 63) // 64), S, x)
    # addPrimes
    P = E.poly(x, S)
    E.add_primes([P], S, ch.special)
    ref = x.copy(); O.add_primes(ref, S, ch.special)
    assert equal(P, ref, Sp)
    # breakIntoDigits of the extremes and of the all -1 digits constant
    c = all_minus_one_digits(ch, S)
    for y in (x, const_rows(ch, S, c)):
        digs = E.break_into_digits([E.poly(y, S)], S)[0]
        rd = O.break_into_digits(y, S)
        assert len(digs) == rd.shape[0] == 8
        assert all(equal(digs[d], rd[d], Sp) for d in range(8))
    # scaleDownToSet: the special primes and two ctxt primes dropped, from extremes over S | special
    QP = ch.product(Sp)
    pat = [0, 1, QP - 1, QP // 2, QP // 2 + 1, (QP - 1) // 2, QP - 2, QP // 2 - 1]
    vals = [pat[j % len(pat)] for j in range(ch.phim)]
    z = O.zeros()
    O.fft_bigpoly(orc.ints_to_limbs(vals, (QP.bit_length() + 63) // 64), Sp, z)
    for p in (1, 2, 257):
        for keep in (S, S[:-2]):
            Z = E.poly(z, Sp)
            E.scale_down([Z], Sp, keep, p)
            ref = z.copy(); O.scale_down(ref, Sp, keep, p)
            assert equal(Z, ref, keep), (p, len(keep))


# ---- linear maps

def units(m, n):
    """The first n units of Z/mZ after 1."""
    return [t for t in range(2, m) if math.gcd(t, m) == 1][:n]


def linmap_case(lib, m, nitems, ks, nd, accumulate=True):
    """hb_hoisted_linear_map where every reduced inner product is q-1 and every constant q-1, so each term of the outer
    128-bit sum is (q-1)^2, the largest a product of reduced values can be: the digits and c0 are q-1 and the keys
    a_0 = nd, b_0 = nd - P (P mod q on the rows of S, 0 on the special rows), every other key q-1, so that
    P*c0 + sum_i D_i*b_i = -1 = sum_i D_i*a_i while the inner sums stay near their own maximum."""
    ch, O, E = small_chain(lib, m, nd=nd) if m & (m - 1) == 0 else top_chain(lib, m, 2, "gen", [1] * nd, 2)
    X = O if O is not None else GenOracle(ch)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    P = ch.product(ch.special)
    ea = np.stack([top(ch, Sp) for _ in range(nd)])
    eb = ea.copy()
    for r in Sp:
        q = ch.primes[r]
        ea[0][r] = nd % q
        eb[0][r] = (nd - (P if r in S else 0)) % q
    dig = np.stack([top(ch, Sp) for _ in range(nd)])
    c0, c1 = top(ch, S), alternating(ch, S)
    cs = top(ch, Sp)
    EA = [E.poly(ea[i], Sp) for i in range(nd)]
    EB = [E.poly(eb[i], Sp) for i in range(nd)]
    CS = E.poly(cs, Sp)
    D = [[E.poly(dig[i], Sp) for i in range(nd)] for _ in range(nitems)]
    C0 = [E.poly(c0, S) for _ in range(nitems)]
    C1 = [E.poly(c1, S) for _ in range(nitems)]
    A0 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    A1 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    E.profile(True)
    E.hoisted_linear_map(D, S, C0, C1, ks, [CS] * len(ks), [None if k == 1 else EA for k in ks], [None if k == 1 else EB for k in ks],
                         A0, A1, accumulate=accumulate)
    E.profile(False)
    assert "k_ks_linmap" in kernels(E), kernels(E)
    # the construction: every reduced inner product is -1
    t0, t1 = c0.copy(), X.zeros()
    X.add_primes_and_scale(t0, S, ch.special)
    X.keyswitch_digits(dig, Sp, ea, eb, t0, t1)
    assert all((t0[r] == ch.primes[r] - 1).all() and (t1[r] == ch.primes[r] - 1).all() for r in Sp)
    acc0 = top(ch, Sp) if accumulate else X.zeros()
    r0, r1 = linmap_reference(X, ch, dig, c0, c1, ks, [cs] * len(ks), [ea] * len(ks), [eb] * len(ks), acc0, acc0)
    for it in range(nitems):
        assert equal(A0[it], r0, Sp) and equal(A1[it], r1, Sp), it
    return E


@pytest.mark.parametrize("nitems", [1, 2, 4, 5])
def test_hoisted_linear_map_64_amounts_at_q_minus_one(lib, nitems):
    """64 amounts (HB_LINMAP_MAXAMT, one k_ks_linmap launch), among them k = 1, over 8 digits, 1, 2, 4 and 5 items (NI = 1,
    2, 4 and 4 + 1), accumulating into q-1.  Bound: at most HB_LINMAP_MAXAMT terms below 2^120 plus the accumulator in
    128 bits, "255 fit" (hb_device.cuh:734-737)."""
    u = units(64, 31)
    ks = [1] + [u[j % len(u)] for j in range(62)] + [1]
    E = linmap_case(lib, 64, nitems, ks, 8)
    st = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert st["k_ks_linmap"] == 1, st


def test_hoisted_linear_map_past_the_128_bit_budget(lib):
    """300 amounts of (q-1)^2 each: more than the 256 products a 128-bit sum holds, so the launch cap must split them
    (hb_engine.cu:2348, HB_LINMAP_MAXAMT at hb_device.cuh:737); a cap above 255 overflows and this fails."""
    u = units(64, 31)
    ks = [u[j % len(u)] for j in range(300)]
    linmap_case(lib, 64, 2, ks, 2)


def test_hoisted_linear_map_general_m_at_q_minus_one(lib):
    """General m (105, Bluestein rows) with primes at the top of the range: 64 amounts, 3 items."""
    u = units(105, 20)
    ks = [1] + [u[j % len(u)] for j in range(63)]
    linmap_case(lib, 105, 3, ks, 3)


def bsgs_setup(lib, m, nd, p=257):
    if m & (m - 1) == 0:
        ch, O, E = top_chain(lib, m, p, "gen", [1] * nd, 2)
        return ch, PowOps(O, ch), E
    ch, O, E = top_chain(lib, m, 2, "gen", [1] * nd, 2)
    return ch, GenOps(ch, [po.cmod_root(q, m) for q in ch.primes]), E


def run_bsgs(ch, X, E, b0, b1, cs, ks, ea, eb, extended, accumulate=True, nitems=1):
    """b0/b1: one list of baby steps shared by every item; cs[t][b]: arrays; ea/eb: one matrix for every giant step."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    R = Sp if extended else S
    nd = len(ch.digits)
    B0 = [E.poly(x, R) for x in b0]
    B1 = [E.poly(x, R) for x in b1]
    CS = [[E.poly(x, R) for x in row] for row in cs]
    EA = [E.poly(ea[i], Sp) for i in range(nd)]
    EB = [E.poly(eb[i], Sp) for i in range(nd)]
    A0 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    A1 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    E.profile(True)
    E.bsgs_linear_map([B0] * nitems, [B1] * nitems, S, ks, CS, [None if k == 1 else EA for k in ks],
                      [None if k == 1 else EB for k in ks], A0, A1, extended=extended, ptxt_space=ptxt(ch), accumulate=accumulate)
    E.profile(False)
    acc = top(ch, Sp) if accumulate else X.zeros()
    r0, r1 = bsgs_reference(X, ch, b0, b1, cs, ks, None, extended, [ea] * len(ks), [eb] * len(ks), acc, acc)
    for it in range(nitems):
        assert equal(A0[it], r0, Sp) and equal(A1[it], r1, Sp), it
    return {r["kernel"]: r["launches"] for r in E.profile_results()}


@pytest.mark.parametrize("extended", [0, 1], ids=["native", "extended"])
@pytest.mark.parametrize("nitems", [1, 2, 4])
def test_bsgs_baby_steps_at_the_launch_cap(lib, nitems, extended):
    """300 baby steps of q-1 times constants of q-1: every product of k_bsgs_mac is (q-1)^2, and the host's cap nbl
    (hb_engine.cu:2439: 128 baby steps for NI = 1 and 4, 240 = HB_BSGS_MAXBABY for NI = 2) must keep each 128-bit sum
    below 256 products (hb_device.cuh:814-819).  A cap past 256 overflows and this fails."""
    ch, X, E = bsgs_setup(lib, 64, 2)
    R = sorted(ch.ctxt + ch.special) if extended else ch.ctxt
    nb = 300
    b0 = [top(ch, R) for _ in range(nb)]
    b1 = [alternating(ch, R) if j % 7 == 3 else top(ch, R) for j in range(nb)]
    cs = [[top(ch, R) for _ in range(nb)] for _ in range(2)]
    ea = top_keys(ch, E)[0]
    st = run_bsgs(ch, X, E, b0, b1, cs, [1, 5], ea, ea, extended, nitems=nitems)
    assert st["k_bsgs_mac"] >= 2 and "k_ks_giant" in st, st


@pytest.mark.parametrize("extended", [0, 1], ids=["native", "extended"])
def test_bsgs_giant_steps_at_the_launch_cap(lib, extended):
    """8 digits and 33 rotated giant steps of one item: a group holds 32 terms and k_ks_giant takes at most
    254/(nd+1) = 28 of them per launch (bsgs_tmax, hb_engine.cu:2427-2429) so that nt*(nd+1) + 1 <= 255 products stay in
    128 bits (hb_device.cuh:890).  Every rotated sum is x0 = -1, x1 = c with digits all -1 (extended form: P*(-1) and
    P*c before the mod-down, whose delta is 0), keys and accumulators are q-1: each term adds P*(q-1) + 8 (q-1)^2 to acc0.
    Without the 254/(nd+1) term the launch takes 32 terms, overflows and this fails."""
    ch, X, E = bsgs_setup(lib, 64, 8)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    R = Sp if extended else S
    P = ch.product(ch.special) if extended else 1
    c = all_minus_one_digits(ch, S)
    # one baby step: x1 = baby1 * w = (q-1) * (-P c) = P c, x0 = baby0 * w = -P
    w, b0 = dense(ch), dense(ch)
    for r in R:
        q = ch.primes[r]
        w[r] = -P * c % q
        b0[r] = (-P * pow(int(w[r][0]), -1, q)) % q if w[r][0] else q - 1
    ks = [u for u in units(64, 31)] + [3, 5]
    assert len(ks) == 33 and 1 not in ks
    ea = np.stack([top(ch, Sp) for _ in range(8)])
    st = run_bsgs(ch, X, E, [b0], [top(ch, R)], [[w] for _ in ks], ks, ea, ea, extended)
    assert st["k_ks_giant"] >= 2, st


def test_bsgs_general_m_at_q_minus_one(lib):
    """General m (105) with primes at the top of the range: 250 baby steps of q-1 for two items (NI = 2: a 240-step launch
    and a 10-step one), constants of q-1, extended form with p = 2."""
    ch, X, E = bsgs_setup(lib, 105, 2)
    Sp = sorted(ch.ctxt + ch.special)
    nb = 250
    b = [top(ch, Sp) for _ in range(nb)]
    cs = [[top(ch, Sp) for _ in range(nb)], [top(ch, Sp) for _ in range(nb)]]
    ea = np.stack([top(ch, Sp) for _ in range(2)])
    st = run_bsgs(ch, X, E, b, b, cs, [1, 2], ea, ea, 1, nitems=2)
    assert st["k_bsgs_mac"] >= 2, st


def test_block_linear_map_64_inner_amounts_at_q_minus_one(lib):
    """hb_block_linear_map with 64 inner amounts (HB_HOIST_MAXAMT, one k_ks_hoist launch; hb_device.cuh:958-960) whose
    hoisted rotations are all (q-1, q-1) (the keys of linmap_case), blocks and accumulators of q-1, and 17 outer amounts in
    both sets of 2 items: 68 (output, item) pairs, more than one group of 64.  Bounds: k_ks_hoist's HB_MAXDIG + 1 products in
    128 bits (hb_device.cuh:958), the 64 products of (q-1)^2 per outer sum in k_bsgs_mac (:814-819) and k_ks_giant's
    nt*(nd+1) + 1 <= 255 (:890)."""
    from test_block_linear_map import _reference as block_reference
    ch, O, E = top_chain(lib, 64, 17, "gen", [1, 1], 2)
    X = PowOps(O, ch)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, nitems, P = 2, 2, ch.product(ch.special)
    ea = np.stack([top(ch, Sp) for _ in range(nd)])
    eb = ea.copy()
    for r in Sp:
        ea[0][r] = nd % ch.primes[r]
        eb[0][r] = (nd - (P if r in S else 0)) % ch.primes[r]
    u = units(64, 31)
    k0 = [1] + [u[j % len(u)] for j in range(63)]
    k1 = [pow(3, j, 64) for j in range(17)]
    kf = pow(3, -17, 64)
    dig, c0, c1 = [top(ch, Sp) for _ in range(nd)], top(ch, S), alternating(ch, S)
    blk = top(ch, Sp)
    cs = [[blk] * len(k1) for _ in k0]
    mats0 = [None if k == 1 else (ea, eb) for k in k0]
    mats1 = [None if k == 1 else (ea, ea) for k in k1]
    EA, EB = [E.poly(ea[i], Sp) for i in range(nd)], [E.poly(eb[i], Sp) for i in range(nd)]
    BLK = E.poly(blk, Sp)
    A0 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    A1 = [E.poly(top(ch, Sp), Sp) for _ in range(nitems)]
    E.profile(True)
    E.block_linear_map([[E.poly(x, Sp) for x in dig] for _ in range(nitems)], S, [E.poly(c0, S)] * nitems, [E.poly(c1, S)] * nitems,
                       k0, [None if m is None else EA for m in mats0], [None if m is None else EB for m in mats0],
                       k1, [None if m is None else EA for m in mats1], [None if m is None else EA for m in mats1],
                       [[BLK] * len(k1) for _ in k0], A0, A1, consts1=[[BLK] * len(k1) for _ in k0], kfinal=kf,
                       evkf_a=EA, evkf_b=EA, ptxt_space=17, accumulate=True)
    E.profile(False)
    st = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert st.get("k_ks_hoist") == 1 and "k_bsgs_mac" in st and "k_ks_giant" in st, st
    r0, r1 = block_reference(X, ch, dig, c0, c1, k0, [None if m is None else m[0] for m in mats0],
                             [None if m is None else m[1] for m in mats0], k1, [None if m is None else ea for m in mats1],
                             [None if m is None else ea for m in mats1], cs, cs, kf, ea, ea, top(ch, Sp), top(ch, Sp))
    for it in range(nitems):
        assert equal(A0[it], r0, Sp) and equal(A1[it], r1, Sp), it
