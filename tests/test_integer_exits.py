"""The kernels that leave RNS, against exact references at the edges of their ranges.

hb_to_poly (k_crt), hb_to_poly_mod_p (k_crt_modp, the tail of SecKey::Decrypt), hb_dcrt_to_powerful (k_pw_scatter,
k_pw_reduce once per factor of m, k_pw_gather, k_crt) and hb_raw_mod_switch (the same powerful-basis rows, then
k_raw_mod_switch, where recryption starts) each round a CRT value to an integer.  A result one multiple of Q off is wrong
in every bit that matters: with p = 2 it flips the decrypted bit, because Q is odd.  Random residues almost never land
where the rounding is decided, so every value here is planted in the basis the kernel rounds in:
  * 0, +-1, +-(Q-1)/2 and its neighbours, Q//2 +- 1, -1 mod Q, and the 4n-ulp band next to +-(Q-1)/2 where hb_conv_v's
    truncated 0.64 fraction hands the decision to the exact CRT;
  * for the powerful basis, the powerful coefficients themselves: the polynomial uploaded is powerfulToPoly of them;
  * for rawModSwitch, c solved from a chosen Y = c*q - round(c*q/Q)*Q: Y at +-(Q-1)/2, inside the margin band around 0 and
    just outside it, and, for an even p^r, Ys of both signs whose u = Y*Q^-1 mod p^r is the tie p^r/2 in each of those
    regimes; and c whose x = round(c*q/Q) + delta lands on +-q/2, +-(q/2 + 1) and up to p^r/2 beyond (the wrap mod q),
    for odd and even q up to the largest admissible q below 2^54.
The rest of every row is uniformly random, so the planted values share a launch with ordinary ones.  Every expected
value is big-integer Python restating the reference (src/DoubleCRT.cpp toPoly, src/keys.cpp:1381-1399 PolyRed,
src/powerful.cpp, src/Ctxt.cpp:2990-3036).  The chains are the largest primes below 2^60, of up to 64 primes (the
HB_MAXROWS cap of the conversions and the per-thread y[HB_MAXROWS] arrays); 65 are refused before anything launches.
The launch profile names the kernels each case is about, and where hb_conv_v decides (k_crt_modp, k_raw_mod_switch) the
engine's exact-fallback counter shows the exact path ran; k_crt reconstructs every coefficient exactly, with no
fallback to count.  Every body runs on the CPU simulator build and, marked gpu, on the H100.
"""
import gc
import math
import random
from fractions import Fraction

import numpy as np
import pytest

import pyoracle as po
from helib_b200.engine import Engine, HbError
from test_norms import from_limbs, to_limbs
from test_value_ranges import R17, kernels, largest_primes, top_chain, transform_divisor

HB_ERR_UNSUPPORTED = -6
QCAP = 1 << 54
PTXT = [2, 4, 256, 3, 257]


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


# ---- rings and chains of the largest primes below 2^60

MVEC = {"105": [3, 5, 7], "45": [9, 5], "4096": None, "R17": None}
CASES = [pytest.param(name, n, id=f"m{name}-n{n}") for name, n in
         [("105", 1), ("105", 2), ("105", 17), ("105", 64), ("45", 1), ("45", 2), ("45", 17), ("45", 64),
          ("4096", 2), ("4096", 64), ("R17", 4)]]


def r17_primes():
    """Two shift-form and two generic largest primes for m = 2^17: the register inverse transforms in both modulus views
    feed k_crt and k_raw_mod_switch."""
    return largest_primes("sp", 2, R17) + largest_primes("gen", 2, R17)


@pytest.fixture
def ring(lib):
    """ring(name, n) -> (engine, idx, Q) on n of the largest primes (general m: the non-trivial powerful basis MVEC[name]
    set).  The engines are closed when the test ends."""
    engines = []

    def make(name, n):
        if name == "R17":
            primes = r17_primes()
            E = Engine(R17, primes, [po.find_psi(q, R17) for q in primes], lib=lib)
        else:
            ch, _, E = top_chain(lib, int(name), 2, "gen", [n], 1)
            primes = ch.primes
        engines.append(E)
        assert len(primes) >= n and all((q - 1) % transform_divisor(E.m) == 0 for q in primes)
        if MVEC[name]:
            E.set_powerful(MVEC[name])
        return E, list(range(n)), math.prod(primes[:n])
    yield make
    gc.collect()
    for E in engines:
        E.close()


_IX = {}


def indexes(mvec):
    """PowerfulIndexes once per factorisation ([5, 17, 257] takes about 9 s)."""
    if mvec is None:
        return None
    key = tuple(mvec)
    if key not in _IX:
        _IX[key] = po.PowerfulIndexes(mvec)
    return _IX[key]


def powerful_to_poly_mod(ix, w, Q):
    """pyoracle.powerful_to_poly(ix, w) mod Q: the same scatter, then the remainder modulo Phi_m over the non-zero
    coefficients of Phi_m only (the dense remainder in Python takes minutes at m = 21845).  Trivial basis: w itself."""
    if ix is None:
        return [c % Q for c in w]
    tmp = np.zeros(ix.m, dtype=object)
    for i, c in enumerate(w):
        tmp[ix.cube_to_poly[ix.short_to_long[i]]] = c % Q
    d = ix.phim
    nz = np.nonzero(np.array(ix.phimx))[0]
    b = np.array(ix.phimx, dtype=object)[nz]
    for i in range(ix.m - 1, d - 1, -1):
        c = tmp[i]
        if c:
            tmp[i - d + nz] -= c * b
    return [int(v) % Q for v in tmp[:d]]


def upload(E, idx, coeffs):
    """A Poly holding the integer polynomial coeffs on the rows idx (hb_poly_from_limbs reduces it modulo every prime)."""
    P = E.poly()
    E.from_limbs([P], idx, [to_limbs(coeffs)])
    return P


def upload_powerful(E, idx, ix, w, Q):
    """A Poly whose powerful-basis coefficients are w mod Q, after checking the reference's own round trip:
    polyToPowerful of the uploaded polynomial gives w back."""
    f = powerful_to_poly_mod(ix, w, Q)
    if ix is not None:
        assert [po.bal(c, Q) for c in po.poly_to_powerful(ix, f)] == [po.bal(c, Q) for c in w]
    return upload(E, idx, f)


def first_diff(got, want, inputs):
    for k, (g, w) in enumerate(zip(got, want)):
        if g != w:
            return {"k": k, "input": inputs[k], "got": g, "want": w}
    return None


# ---- planted values

def band(n):
    """Offsets j <= 4n from +-(Q-1)/2 (the margin of the truncated fraction is 4n ulps): the ends and a few between."""
    return sorted({0, 1, 2, 3, 2 * n, 4 * n - 1, 4 * n})


def extremes(M, n):
    A = (M - 1) // 2
    vals = [0, 1, -1, 2, -2, A, -A, A - 1, -A + 1, A + 1, -A - 1, A - 2, -A + 2, M // 2 + 1, M // 2 - 1, M - 1,
            M // 3, -(M // 3)]
    return vals + [-A + j for j in band(n)] + [A - j for j in band(n)]


def rows_with(plants, N, M, rnd):
    """Rows of N coefficients, each holding at most 3N/4 of the planted values at random places among uniformly random
    ones mod M."""
    per = max(1, 3 * N // 4)
    out = []
    for k in range(0, len(plants), per):
        chunk = plants[k:k + per]
        f = [rnd.randrange(M) for _ in range(N)]
        for pos, v in zip(rnd.sample(range(N), len(chunk)), chunk):
            f[pos] = v
        out.append(f)
    return out


def unit(p2r):
    """A unit mod p^r other than 1 (p^r = 2 has none)."""
    return next((t for t in range(p2r // 2 + 1, p2r) if math.gcd(t, p2r) == 1), 1)


# ---- rawModSwitch

def raw_ms_ref(c, Q, q, p2r):
    """Ctxt::rawModSwitch of one balanced powerful coefficient c (src/Ctxt.cpp:2990-3036) -> (x, x before the reduction
    mod q, Y, delta).  Ties at x = +-q/2 of an even q stay (the reference flips a coin there); a tie of an even p^r at
    Y = 0 cannot occur, because delta = 0 there."""
    X, Y = divmod(c * q, Q)
    if Y > Q // 2:
        Y -= Q
        X += 1
    delta = (Y % p2r) * pow(Q, -1, p2r) % p2r
    assert not (Y == 0 and delta)
    if delta > p2r // 2 or (p2r % 2 == 0 and delta == p2r // 2 and Y < 0):
        delta -= p2r
    x = X + delta
    assert abs(Fraction(c * q, Q) - x) <= Fraction(p2r, 2), (c, x)        # the reference's sanity check (:3021-3030)
    xw = x
    if xw > q // 2:
        xw -= q
    elif xw < -(q // 2):
        xw += q
    ctarget = c * q * pow(Q, -1, p2r)
    assert any((xw + k * q - ctarget) % p2r == 0 for k in (-1, 0, 1)), (c, xw)   # x = c*q*Q^-1 (mod p^r), one q wrap
    return xw, x, Y, delta


def moduli(p2r, Q):
    """q = p^e + 1 for a small and for the largest e below the 2^54 cap (odd for p = 2, even for odd p), and the largest
    admissible q below 2^54: coprime to p^r and to Q (for p = 2, 2^54 - 1 = 3^4 7 19 73 87211 262657: none of those
    divides Q)."""
    p = 2 if p2r % 2 == 0 else p2r
    e = 1
    while p ** (e + 1) + 1 < QCAP:
        e += 1
    small = next(p ** k + 1 for k in range(1, e + 1) if p ** k >= 1 << 11)
    top = QCAP - 1
    while math.gcd(top, p2r) != 1 or math.gcd(top, Q) != 1:
        top -= 1
    out = [small, p ** e + 1, top]
    assert all(1 < q < QCAP and math.gcd(q, p2r) == 1 and math.gcd(q, Q) == 1 for q in out)
    return out


def plant_x(T, Q, q, p2r):
    """A balanced c whose value before the reduction mod q is T, or None when no c reaches T: c*q = X0*Q + Y with
    X0 = T - delta, Y = -X0*Q (mod q) and Y = delta*Q (mod p^r), |Y| <= (Q-1)/2."""
    A, M, h = (Q - 1) // 2, q * p2r, p2r // 2
    qinv = pow(q, -1, p2r)
    for delta in range(-h, h + 1):
        X0 = T - delta
        a, b = (-X0 * Q) % q, (delta * Q) % p2r
        Y0 = a + q * ((b - a) * qinv % p2r)
        for s in (1, -1):
            k = (s * (Q // 4) - Y0) // M
            for Y in (Y0 + M * k, Y0 + M * (k + 1)):
                if abs(Y) > A:
                    continue
                c = (X0 * Q + Y) // q
                if abs(c) <= A and raw_ms_ref(c, Q, q, p2r)[1] == T:
                    return c
    return None


def ms_plants(Q, q, p2r, n):
    """The balanced c of a rawModSwitch case: the extremes of c, c solved from chosen Y, and c landing on the wrap."""
    A = (Q - 1) // 2
    B = 4 * n * Q >> 64                       # |Y| <= B: inside the 4n-ulp margin band around 0
    Ys = [A, A - 1, A - 2, 1, 2, 3, 5, B + 1, B + 2, 2 * B + 3] + ([B, B - 1] if B > 8 else [])
    if p2r % 2 == 0:                          # ties: Y = p^r/2 (mod p^r) (Q is odd)
        t = p2r // 2

        def up(y):
            return y + (t - y) % p2r

        def down(y):
            return y - (y - t) % p2r
        Ys += [down(A), up(-A), t, t - p2r, t + p2r, t - 2 * p2r, up(B + 1), down(-B - 1)]
        if B > 2 * p2r:
            Ys += [down(B), up(-B)]
    Ys += [-y for y in Ys]
    qi = pow(q, -1, Q)
    plants = extremes(Q, n) + [po.bal(Y * qi, Q) for Y in Ys]
    for Y in Ys:                              # c*q = Y (mod Q), and the reference reads that Y back
        assert raw_ms_ref(po.bal(Y * qi, Q), Q, q, p2r)[2] == Y
    qh = q // 2
    for T in (qh, -qh, qh + 1, -qh - 1, qh + p2r // 2, -qh - p2r // 2, qh - 1, -qh + 1):
        c = plant_x(T, Q, q, p2r)
        assert c is not None or q * p2r > Q // 4, T      # always reachable unless q*p^r is close to Q
        if c is not None:
            plants.append(c)
    return plants


def check_plants(plants, Q, q, p2r):
    """The planted values reach what they are for: both wrap directions, and for an even p^r ties of both signs."""
    refs = [raw_ms_ref(po.bal(c, Q), Q, q, p2r) for c in plants]
    qh = q // 2
    assert any(x > qh for _, x, _, _ in refs) and any(x < -qh for _, x, _, _ in refs)
    if q % 2 == 0:
        assert any(x == qh for _, x, _, _ in refs) and any(x == -qh for _, x, _, _ in refs)
    if p2r % 2 == 0:
        ties = [Y for _, _, Y, d in refs if abs(d) == p2r // 2]
        assert any(Y > 0 for Y in ties) and any(Y < 0 for Y in ties)


# ---- a. toPoly and the decryption tail

@pytest.mark.parametrize("name,n", CASES)
def test_to_poly_and_decryption_tail_at_the_extremes(ring, name, n):
    """hb_to_poly (balanced and positive) must return bal(c, Q) (c mod Q), and hb_to_poly_mod_p (c mod p^r) * factor mod
    p^r with c balanced (PolyRed, include/helib_b200.h), for p^r = 2, 4, 256, 3, 257 and factor 1 and a unit."""
    E, idx, Q = ring(name, n)
    rnd = random.Random(10 + n)
    rows = rows_with(extremes(Q, n), E.N, Q, rnd)
    X = [upload(E, idx, f) for f in rows]
    E.reset_stats()
    E.profile(True)
    for f, P in zip(rows, X):
        want = [po.bal(c, Q) for c in f]
        got = from_limbs(E.to_poly(P, idx))
        assert got == want, first_diff(got, want, f)
        got = from_limbs(E.to_poly(P, idx, positive=True))
        assert got == [c % Q for c in f], first_diff(got, [c % Q for c in f], f)
        for p2r in PTXT:
            for factor in sorted({1, unit(p2r)}):
                got = E.to_poly_mod_p(P, idx, p2r, factor).tolist()
                wp = [c % p2r * factor % p2r for c in want]
                assert got == wp, (p2r, factor, first_diff(got, wp, want))
    E.profile(False)
    ran = kernels(E)
    assert {"k_crt", "k_crt_modp"} <= ran, ran
    if name == "R17":
        assert "k1_inv_cols" in ran, ran
    if n >= 2:       # one 60-bit prime: 1/Q is wider than the margin band, so no integer coefficient falls in it
        assert E.stats()["exact_fallbacks"] > 0, E.stats()


# ---- b. the powerful basis

@pytest.mark.parametrize("name,n", CASES)
def test_dcrt_to_powerful_at_the_extremes(ring, name, n):
    """hb_dcrt_to_powerful of the polynomial whose powerful-basis coefficients w are planted must return bal(w, Q); the
    engine's index map must be the reference's."""
    E, idx, Q = ring(name, n)
    ix = indexes(MVEC[name])
    factors, to_poly = E.powerful_info()
    if ix is not None:
        assert factors == MVEC[name]
        assert to_poly.tolist() == [ix.cube_to_poly[ix.short_to_long[i]] for i in range(E.N)]
    else:
        assert len(factors) == 1 and to_poly.tolist() == list(range(E.N))
    rnd = random.Random(20 + n)
    rows = rows_with(extremes(Q, n), E.N, Q, rnd)
    X = [upload_powerful(E, idx, ix, w, Q) for w in rows]
    E.profile(True)
    for w, P in zip(rows, X):
        want = [po.bal(c, Q) for c in w]
        got = from_limbs(E.dcrt_to_powerful(P, idx))
        assert got == want, first_diff(got, want, w)
    E.profile(False)
    ran = kernels(E)
    assert "k_crt" in ran, ran
    if ix is not None:
        assert {"k_pw_scatter", "k_pw_reduce", "k_pw_gather"} <= ran, ran


# ---- c. rawModSwitch

def run_raw_mod_switch(E, idx, Q, ix, q, p2r, rows):
    """hb_raw_mod_switch of every row against raw_ms_ref, coefficient by coefficient, in the powerful basis the ABI
    returns."""
    for w in rows:
        P = upload_powerful(E, idx, ix, w, Q)
        got = E.raw_mod_switch(P, idx, q, p2r).tolist()
        want = [raw_ms_ref(po.bal(c, Q), Q, q, p2r)[0] for c in w]
        assert got == want, (q, p2r, first_diff(got, want, [po.bal(c, Q) for c in w]))


@pytest.mark.parametrize("p2r", PTXT)
@pytest.mark.parametrize("name,n", CASES)
def test_raw_mod_switch_at_its_rounding_boundaries(ring, name, n, p2r):
    """hb_raw_mod_switch for q = p^e + 1 (small and largest e) and the largest admissible q below 2^54: the Y regimes of
    the delta tie, the c extremes of the first rounding and the wrap mod q, against Ctxt::rawModSwitch per coefficient."""
    E, idx, Q = ring(name, n)
    ix = indexes(MVEC[name])
    rnd = random.Random(1000 * n + p2r)
    for q in moduli(p2r, Q):
        plants = ms_plants(Q, q, p2r, n)
        check_plants(plants, Q, q, p2r)
        E.reset_stats()
        E.profile(True)
        run_raw_mod_switch(E, idx, Q, ix, q, p2r, rows_with(plants, E.N, Q, rnd))
        E.profile(False)
        ran = kernels(E)
        assert "k_raw_mod_switch" in ran, ran
        if ix is not None:
            assert "k_pw_reduce" in ran, ran
        if n >= 2:
            assert E.stats()["exact_fallbacks"] > 0, (q, E.stats())


# ---- d. limits

def test_65_source_primes_are_refused_before_anything_runs(ring):
    """HB_MAXROWS = 64 source primes: 65 are refused with HB_ERR_UNSUPPORTED by every entry point that leaves RNS, and
    nothing is launched (the conversion table is built before the first kernel)."""
    E, idx, Q = ring("105", 65)
    X = upload(E, idx, [1] * E.N)
    E.profile(True)
    calls = [lambda: E.to_poly(X, idx), lambda: E.to_poly_mod_p(X, idx, 2), lambda: E.dcrt_to_powerful(X, idx),
             lambda: E.raw_mod_switch(X, idx, (1 << 11) + 1, 2)]
    for call in calls:
        with pytest.raises(HbError) as ei:
            call()
        assert ei.value.code == HB_ERR_UNSUPPORTED, ei.value
    E.profile(False)
    assert E.profile_results() == [], E.profile_results()


def test_raw_mod_switch_refuses_q_from_2_to_the_54(ring):
    """q < 2^54 keeps sum_j k_j and q*v0 in 64 bits (k_raw_mod_switch): 2^54 (with an odd p^r) and 2^54 + 1 (with p^r = 2)
    are refused with HB_ERR_UNSUPPORTED before anything runs."""
    E, idx, Q = ring("105", 2)
    X = upload(E, idx, [1] * E.N)
    E.profile(True)
    for q, p2r in ((QCAP, 3), (QCAP, 257), (QCAP + 1, 2)):
        with pytest.raises(HbError) as ei:
            E.raw_mod_switch(X, idx, q, p2r)
        assert ei.value.code == HB_ERR_UNSUPPORTED, (q, p2r, ei.value)
    E.profile(False)
    assert E.profile_results() == [], E.profile_results()


# ---- e. full-size rings (GPU)

CFG5 = 21845


@pytest.mark.gpu
@pytest.mark.parametrize("chain", ["own", "gen17"])
def test_config5_ring_powerful_basis_and_raw_mod_switch(cuda_lib, chain):
    """Config 5's ring (m = 21845 = 5*17*257, phi = 16384, the ring thin recryption is built for) with the powerful basis
    [5, 17, 257], p^r = 2 and q = 2^11 + 1: on its own chain (buildModChain(21845, 2, 1, 580, 2): 10 ctxt primes) and on
    17 of the largest primes; every coefficient of hb_dcrt_to_powerful and hb_raw_mod_switch against the reference."""
    if chain == "own":
        ch = po.build_mod_chain(CFG5, 2, 1, 580, 2)
        primes, idx = ch.primes, ch.ctxt
        assert len(idx) == 10
    else:
        primes, idx = largest_primes("gen", 17, CFG5), list(range(17))
    E = Engine(CFG5, primes, None, lib=cuda_lib)
    try:
        E.set_powerful([5, 17, 257])
        ix = indexes([5, 17, 257])
        Q, n, q, p2r = math.prod(primes[i] for i in idx), len(idx), (1 << 11) + 1, 2
        plants = ms_plants(Q, q, p2r, n)
        check_plants(plants, Q, q, p2r)
        rnd = random.Random(5 + n)
        [w] = rows_with(plants, E.N, Q, rnd)
        P = upload_powerful(E, idx, ix, w, Q)
        E.reset_stats()
        E.profile(True)
        got = from_limbs(E.dcrt_to_powerful(P, idx))
        want = [po.bal(c, Q) for c in w]
        assert got == want, first_diff(got, want, w)
        got = E.raw_mod_switch(P, idx, q, p2r).tolist()
        want = [raw_ms_ref(c, Q, q, p2r)[0] for c in want]
        assert got == want, first_diff(got, want, [po.bal(c, Q) for c in w])
        E.profile(False)
        assert {"k_pw_reduce", "k_crt", "k_raw_mod_switch"} <= kernels(E), kernels(E)
        assert E.stats()["exact_fallbacks"] > 0, E.stats()
    finally:
        gc.collect()
        E.close()


@pytest.mark.gpu
def test_config3_chain_to_poly_and_decryption_tail(cuda_lib):
    """Config 3's chain (m = 2^17, 26 ctxt primes): hb_to_poly and hb_to_poly_mod_p at p = 2 and 257 with the planted
    extremes among 2^16 coefficients."""
    from common import chain
    ch, psis = chain(1 << 17, 257, 1, 1500, 3)
    E = Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=cuda_lib)
    try:
        idx, Q = ch.ctxt, ch.product(ch.ctxt)
        assert len(idx) == 26
        [f] = rows_with(extremes(Q, len(idx)), E.N, Q, random.Random(3))
        P = upload(E, idx, f)
        E.reset_stats()
        E.profile(True)
        want = [po.bal(c, Q) for c in f]
        got = from_limbs(E.to_poly(P, idx))
        assert got == want, first_diff(got, want, f)
        for p2r, factor in ((2, 1), (257, 1), (257, unit(257))):
            got = E.to_poly_mod_p(P, idx, p2r, factor).tolist()
            wp = [c % p2r * factor % p2r for c in want]
            assert got == wp, (p2r, factor, first_diff(got, wp, want))
        E.profile(False)
        assert {"k_crt", "k_crt_modp"} <= kernels(E), kernels(E)
        assert E.stats()["exact_fallbacks"] > 0, E.stats()
    finally:
        gc.collect()
        E.close()
