"""The canonical-embedding norms against exact references, at the edges of the balanced range.

The norms are the engine's only floating-point outputs, and the Ctxt layer turns them straight into noise bounds: the
digits' norms at every key switch, the mod-down's ||delta/P|| at every modDownToSet.  A norm that comes out too small
makes the bound smaller than the noise.  The conversion kernels (k_conv, k1_conv in both modulus views, k_conv_plain)
hand each coefficient to the norm kernels as x/Q, taken from a 0.64 fixed-point sum that is truncated, so always a little
low; coefficients at -(Q-1)/2 or within the 4n-ulp margin of it reach the exact fallback of hb_conv_v, which must fix the
fraction (-1/2) as well as the integer.  Random residues almost never fall there, so the inputs here are built from exact
integers: the coefficients +-(Q-1)/2 and their neighbours, scattered through random data, then single coefficients,
all-equal polynomials and cosines peaking at a chosen evaluation point for the norm kernels themselves (k_norm_twist /
k_norm_stage, k_gen_norm), batches past one chunk, and the norms of hb_bsgs_linear_map_norm.

Every reference is pyoracle.embedding_largest_coeff of the exact integers (for the mod-down, of delta/P from the exact
delta), and where a closed form exists (c*X^k: |c|; for power-of-two m, c*sum_k X^k: |c|/sin(pi/2N)) that as well.  The
tolerance is 1e-9 relative (1e-9*|ln| for the ln variants) plus the documented floor: each x/Q is off by at most 4n*2^-64,
so a norm by at most 4n*N*2^-64*Q, either way (include/helib_b200.h).  The integer rows stay bit-exact, the engine's
exact-fallback counter shows the band was reached, and the launch profile names the intended kernels.  Every body runs on
the CPU simulator build and, marked gpu, on the H100.
"""
import gc
import math
from fractions import Fraction

import numpy as np
import pytest

import pyoracle as po
from test_bsgs import PowOps, _reference as bsgs_reference
from test_value_ranges import R17, kernels, top_chain, units

P_ODD = 257


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


# ---- rings: one per conversion kernel, three digits of two primes and two special primes, so that every set a
# conversion reads has Q > 2^100 and -(Q-1)/2 lies inside the fallback band

RINGS = {
    "k_conv-64": (64, "gen"),
    "k_conv-4096": (4096, "gen"),
    "k1_conv-sp": (R17, "sp"),          # shift-form primes: k1_conv<true>
    "k1_conv-gen": (R17, "gen"),        # generic modulus view: k1_conv<false>
    "k_conv_plain-105": (105, "gen"),
    "k_conv_plain-1271": (1271, "gen"),  # phi(m) = 1200: k_gen_norm's last tile is 176 wide
}


@pytest.fixture
def ring(lib):
    """ring(name, digit_sizes) -> (chain, oracle, engine).  The engines are closed when the test ends, pass or fail: an
    engine at N = 2^16 holds several hundred MB of device scratch, which would otherwise stay allocated for the rest of
    the session and starve the tests that follow."""
    engines = []

    def make(name, digit_sizes=(2, 2, 2)):
        m, form = RINGS[name]
        ch, O, E = top_chain(lib, m, P_ODD, form, list(digit_sizes), 2)
        engines.append(E)
        return ch, O, E
    yield make
    gc.collect()     # the test's Polys first, while their engine is open
    for E in engines:
        E.close()


def conv_kernel(name):
    return name.split("-")[0]


def norm_kernel(ch):
    return "k_norm_stage" if ch.m & (ch.m - 1) == 0 else "k_gen_norm"


MASK = (1 << 64) - 1


def to_limbs(vals):
    """Two's-complement little-endian limbs [N][L] of Python ints (orc.ints_to_limbs, a column at a time)."""
    L = max(2, max(abs(v) for v in vals).bit_length() // 64 + 2)
    mod = 1 << (64 * L)
    vs = [v % mod for v in vals]
    out = np.empty((len(vs), L), dtype=np.uint64)
    for l in range(L):
        out[:, l] = np.array([(v >> (64 * l)) & MASK for v in vs], dtype=np.uint64)
    return out


def from_limbs(a):
    """orc.limbs_to_ints, a column at a time."""
    N, L = a.shape
    cols = [a[:, l].tolist() for l in range(L)]
    out = []
    for k in range(N):
        v = 0
        for l in range(L - 1, -1, -1):
            v = (v << 64) | cols[l][k]
        out.append(v - (1 << (64 * L)) if cols[L - 1][k] >> 63 else v)
    return out


def rows_of(ch, O, coeffs, idx):
    """The evaluation rows idx of the integer polynomial coeffs, exact: the oracle's transforms for power-of-two m,
    pyoracle's definition-level Bluestein DFT otherwise."""
    out = np.zeros((len(ch.primes), ch.phim), dtype=np.uint64)
    if O is not None:
        O.fft_bigpoly(to_limbs(coeffs), idx, out)
        return out
    for i in idx:
        q = ch.primes[i]
        out[i] = np.array(po.gen_fft([c % q for c in coeffs], q, ch.m, po.cmod_root(q, ch.m)), dtype=np.uint64)
    return out


def upload(ch, O, E, coeffs, idx):
    """A Poly holding coeffs on the rows idx.  For general m the engine reduces the coefficients itself (hb_poly_from_limbs,
    pinned against pyoracle in test_general_m): the definition-level DFT in Python is the slow part of these tests."""
    if O is not None:
        return E.poly(rows_of(ch, O, coeffs, idx), idx)
    P = E.poly()
    E.from_limbs([P], idx, [to_limbs(coeffs)])
    return P


def checked_rows(ch, idx):
    """The rows an integer result is compared on: all of them, but for general m with phi(m) > 1000 the first and the
    last, each against pyoracle's DFT."""
    return list(idx) if ch.m & (ch.m - 1) == 0 or ch.phim <= 1000 else [idx[0], idx[-1]]


def equal(P, ch, O, coeffs, idx):
    """P's rows idx are those of the integer polynomial coeffs, bit for bit."""
    idx = checked_rows(ch, idx)
    return bool((P.download(idx)[idx] == rows_of(ch, O, coeffs, idx)[idx]).all())


# ---- references and tolerances

def ref_ln(coeffs, m):
    if not any(coeffs):
        return -math.inf
    mant, shift = po.embedding_largest_coeff(coeffs, m)
    return math.log(mant) + shift * math.log(2.0)


def ref_norm_float(vals, m):
    """embeddingLargestCoeff of a polynomial with real coefficients (delta/P), as the reference evaluates it."""
    N = len(vals)
    if m & (m - 1) == 0:
        k = np.arange(N)
        return float(np.max(np.abs(np.fft.ifft(np.array(vals) * np.exp(1j * np.pi * k / N)) * N)))
    ff = np.zeros(m)
    ff[:N] = vals
    v = np.fft.fft(ff)
    return float(np.max(np.abs(v[[i for i in range(1, m // 2 + 1) if math.gcd(i, m) == 1]])))


def ln_floor(N, n, Q):
    """ln of the norm's error bound 4n*N*2^-64*Q for x/Q over n source primes."""
    return math.log(4 * n * N) - 64 * math.log(2.0) + math.log(Q) if Q > 1 else -math.inf


def assert_ln(got, want, floor, what):
    """|norm - ref| within 1e-9*|ln ref| (relative, in ln) plus the floor; all three given as ln."""
    if want == -math.inf and floor == -math.inf:
        assert got == -math.inf, (what, got)
        return
    s = max(want, floor)
    g, w, f = math.exp(got - s), math.exp(want - s), math.exp(floor - s)
    t = 1e-9 * abs(want) if want > -math.inf else 0.0
    assert w * math.exp(-t) - f <= g <= w * math.exp(t) + f, (what, got, want, floor)


def assert_norm(got, want, floor, what):
    assert abs(got - want) <= 1e-9 * want + floor, (what, got, want, floor)


# ---- the exact operations the entry points restate

def bgv_delta(x, Pd, p):
    """scaleDownToSet's delta (src/DoubleCRT.cpp:1485-1511): x mod P balanced, then the multiple of P that makes it
    divisible by p, the tie of an even p read from the sign of x mod P."""
    d = po.bal(x, Pd)
    if p == 1:
        return d
    u = d % p
    if u:
        u = u * pow(Pd % p, -1, p) % p
        if u > p // 2 or (p % 2 == 0 and u == p // 2 and d < 0):
            u -= p
        d -= Pd * u
    return d


def digits_of(ch, x, S):
    """breakIntoDigits' balanced mixed-radix digits of x over the digits of S.  A digit S has no prime of is the zero
    polynomial, and the later digits are still divided by its full product (src/DoubleCRT.cpp:551-556)."""
    out = []
    for t, dg in enumerate(ch.digits):
        part = [i for i in dg if i in S]
        Qd = ch.product(part)
        if not part:
            out.append([0] * len(x))
            rest = ch.product([i for d in ch.digits[t + 1:] for i in d if i in S])
            inv = pow(ch.product(dg), -1, rest) if rest > 1 else 0
            x = [po.bal(c * inv, rest) for c in x]
            continue
        e = [po.bal(c, Qd) for c in x]
        out.append(e)
        x = [(c - ec) // Qd for c, ec in zip(x, e)]
    return out


# ---- patterns at the edges of the balanced range of M (n source primes)

PATTERNS = ["table", "band", "plusA", "scatter"]


def uniform(M, N, rng):
    """N uniformly random balanced residues mod M, none of them at -(M-1)/2."""
    A = (M - 1) // 2
    return [c if c != -A else 0 for c in (po.bal(int.from_bytes(rng.bytes(M.bit_length() // 8 + 8), "little"), M) for _ in range(N))]


def pattern(kind, M, N, n, rng):
    """(coefficients, how many of them sit in the fallback band).  A = (M-1)/2, B = A//2:
    'table' -A - B X - B X^2; 'band' -A + j for j <= 4n; 'plusA' A - j for j <= 4n (the band's other side, where the
    truncated sum rounds correctly); 'scatter' -A at random places in uniformly random data."""
    A, B = (M - 1) // 2, (M - 1) // 4
    f = [0] * N
    if kind == "table":
        f[:3] = [-A, -B, -B]
        return f, 1
    if kind == "band":
        f[:4 * n + 1] = [-A + j for j in range(4 * n + 1)]
        return f, 4 * n + 1
    if kind == "plusA":
        f[:4 * n + 1] = [A - j for j in range(4 * n + 1)]
        return f, 4 * n + 1
    assert kind == "scatter"
    f = uniform(M, N, rng)
    pos = rng.choice(N, size=max(3, N // 16), replace=False)
    for k in pos:
        f[int(k)] = -A
    return f, len(pos)


# ---- a. balanced-range extremes on every conversion kernel

@pytest.mark.parametrize("name", list(RINGS))
def test_add_primes_norm_at_the_balanced_extremes(ring, name):
    """hb_add_primes_norm from the six ctxt primes to the special primes, one item per pattern."""
    ch, O, E = ring(name)
    rng = np.random.default_rng(1)
    S, N = ch.ctxt, ch.phim
    Q = ch.product(S)
    pats = [pattern(k, Q, N, len(S), rng) for k in PATTERNS]
    X = [upload(ch, O, E, f, S) for f, _ in pats]
    E.reset_stats()
    E.profile(True)
    got = E.add_primes_norm(X, S, ch.special)
    E.profile(False)
    assert E.stats()["exact_fallbacks"] >= sum(b for _, b in pats), E.stats()
    assert {conv_kernel(name), norm_kernel(ch)} <= kernels(E), kernels(E)
    fl = ln_floor(N, len(S), Q)
    for kind, (f, _), P, g in zip(PATTERNS, pats, X, got):
        assert equal(P, ch, O, f, ch.special), kind
        assert_ln(g, ref_ln(f, ch.m), fl, kind)


@pytest.mark.parametrize("name", list(RINGS))
def test_break_into_digits_norm_with_each_digit_at_the_extremes(ring, name):
    """hb_break_into_digits_norm of x = sum_i d_i Q_0..Q_(i-1) with balanced digits d_i: item (i, pattern) has digit i at
    the pattern over Q_i and the other digits uniformly random, so each digit's conversion meets -(Q_i-1)/2 in turn."""
    ch, O, E = ring(name)
    rng = np.random.default_rng(2)
    S, Sp, N = ch.ctxt, sorted(ch.ctxt + ch.special), ch.phim
    Qd = [ch.product(d) for d in ch.digits]
    items, nband = [], 0
    for i in range(len(ch.digits)):
        for kind in PATTERNS if N < 1 << 16 else PATTERNS[:2]:    # at N = 2^16 the Python side dominates: two patterns
            digs = [uniform(q, N, rng) for q in Qd]
            digs[i], b = pattern(kind, Qd[i], N, len(ch.digits[i]), rng)
            nband += b
            x, scale = [0] * N, 1
            for d, q in zip(digs, Qd):
                x = [a + c * scale for a, c in zip(x, d)]
                scale *= q
            assert digits_of(ch, x, S) == digs
            items.append((i, kind, x, digs))
    X = [upload(ch, O, E, x, S) for _, _, x, _ in items]
    E.reset_stats()
    E.profile(True)
    D, got = E.break_into_digits_norm(X, S)
    E.profile(False)
    assert E.stats()["exact_fallbacks"] >= nband, E.stats()
    assert {conv_kernel(name), norm_kernel(ch)} <= kernels(E), kernels(E)
    for it, (i, kind, x, digs) in enumerate(items):
        for d, (dd, q) in enumerate(zip(digs, Qd)):
            assert equal(D[it][d], ch, O, dd, Sp), (i, kind, d)
            assert_ln(got[it, d], ref_ln(dd, ch.m), ln_floor(N, len(ch.digits[d]), q), (i, kind, d))


@pytest.mark.parametrize("p", [1, P_ODD, 2])
@pytest.mark.parametrize("name", list(RINGS))
def test_scale_down_norm_at_the_balanced_extremes(ring, name, p):
    """hb_scale_down_norm dropping the special primes, with x mod P at the patterns over P and x = delta0 + P*r, r
    uniformly random: ptxt 1 (CKKS), an odd p and the even 2, whose tie rule reads the sign of x mod P."""
    ch, O, E = ring(name)
    rng = np.random.default_rng(3 + p)
    S, Sp, N = ch.ctxt, sorted(ch.ctxt + ch.special), ch.phim
    Pd, Q = ch.product(ch.special), ch.product(S)
    items, nband = [], 0
    for kind in PATTERNS:
        d0, b = pattern(kind, Pd, N, len(ch.special), rng)
        r = uniform(Q, N, rng)
        x = [a + Pd * c for a, c in zip(d0, r)]
        nband += b
        items.append((kind, x))
    X = [upload(ch, O, E, x, Sp) for _, x in items]
    E.reset_stats()
    E.profile(True)
    got = E.scale_down_norm(X, Sp, S, p)
    E.profile(False)
    assert E.stats()["exact_fallbacks"] >= nband, E.stats()
    assert {conv_kernel(name), norm_kernel(ch)} <= kernels(E), kernels(E)
    fl = 4 * len(ch.special) * N * 2.0 ** -64
    for (kind, x), P, g in zip(items, X, got):
        delta = [bgv_delta(c, Pd, p) for c in x]
        if O is not None:     # the oracle's own delta
            assert from_limbs(O.scale_down(rows_of(ch, O, x, Sp), Sp, S, p, want_delta=True)) == delta, kind
        assert equal(P, ch, O, [(c - d) // Pd for c, d in zip(x, delta)], S), kind
        want = ref_norm_float([float(Fraction(d, Pd)) for d in delta], ch.m)
        assert_norm(g, want, fl, kind)


# ---- b. the floor

@pytest.mark.parametrize("name", ["k_conv-64", "k1_conv-sp", "k_conv_plain-105", "k_conv_plain-1271"])
def test_small_polynomials_get_at_most_the_floor(ring, name):
    """Coefficients far below 2^-40 Q: c X^k for c = 1, -1, 3 and 2^70 over the full ctxt set (addPrimes) and over the
    digits (breakIntoDigits, where c lies in digit 0 and the other digits are the zero polynomial over a non-empty set:
    -inf).  Each norm lies within 4n*N*2^-64*Q of |c|, on either side; the zero polynomial's is 0 (ln -inf) over the
    ctxt set as well.  None of these coefficients reaches the fallback band."""
    ch, O, E = ring(name)
    S, Sp, N = ch.ctxt, sorted(ch.ctxt + ch.special), ch.phim
    Q = ch.product(S)
    cases = [(1, 0), (-1, 5), (3, N - 1), (1 << 70, 1), (0, 0)]
    polys = []
    for c, k in cases:
        f = [0] * N
        f[k] = c
        polys.append(f)
    X = [upload(ch, O, E, f, S) for f in polys]
    E.reset_stats()
    got = E.add_primes_norm(X, S, ch.special)
    for (c, k), f, P, g in zip(cases, polys, X, got):
        want = math.log(abs(c)) if c else -math.inf
        assert abs(want - ref_ln(f, ch.m)) <= 1e-12 if c else ref_ln(f, ch.m) == want
        if c:
            assert_ln(g, want, ln_floor(N, len(S), Q), (c, k))
        else:
            assert g == -math.inf
        assert equal(P, ch, O, f, ch.special), (c, k)
    X = [upload(ch, O, E, f, S) for f in polys]
    D, got = E.break_into_digits_norm(X, S)
    assert E.stats()["exact_fallbacks"] == 0, E.stats()
    for it, (c, k) in enumerate(cases):
        assert_ln(got[it, 0], math.log(abs(c)) if c else -math.inf, ln_floor(N, len(ch.digits[0]), ch.product(ch.digits[0])) if c else -math.inf, (c, k))
        for d in range(1, len(ch.digits)):
            assert got[it, d] == -math.inf, (c, k, d)
        assert equal(D[it][0], ch, O, polys[it], Sp)


# ---- c. the norm kernels themselves

def evaluations(f, m):
    """|f| at every evaluation point the norm takes the max over, in the reference's order: zeta^(2j+1) for power-of-two
    m, W^i for i in Z_m^*, i <= m/2 otherwise."""
    N = len(f)
    ff = np.array([float(c) for c in f])
    if m & (m - 1) == 0:
        k = np.arange(N)
        return list(range(N)), np.abs(np.fft.ifft(ff * np.exp(1j * np.pi * k / N)) * N)
    pts = [i for i in range(1, m // 2 + 1) if math.gcd(i, m) == 1]
    full = np.zeros(m)
    full[:N] = ff
    return pts, np.abs(np.fft.fft(full)[pts])


def peaked(ch, C):
    """(label, coefficients, evaluation point of the largest value or None, closed-form norm or None): cosines peaking at
    chosen evaluation points (a real polynomial takes the same value at the conjugate point too), single coefficients at
    k = 0 and N-1, the all-equal polynomial."""
    N, m = ch.phim, ch.m
    out = []
    if m & (m - 1) == 0:
        for j0 in (0, N // 4, N // 2, N - 1):     # f(zeta^(2 j0 + 1)) = C N / 2, and at the conjugate point N-1-j0
            out.append((f"cos-{j0}", [round(C * math.cos(math.pi * k * (2 * j0 + 1) / N)) for k in range(N)], j0, None))
        out.append(("equal", [C] * N, None, C / math.sin(math.pi / (2 * N))))
    else:
        pts = [i for i in range(1, m // 2 + 1) if math.gcd(i, m) == 1]
        for i0 in (pts[0], pts[-1]):
            out.append((f"cos-{i0}", [round(C * math.cos(2 * math.pi * i0 * k / m)) for k in range(N)], i0, None))
        out.append(("equal", [C] * N, None, None))
    out.append(("X^0", [C] + [0] * (N - 1), None, C))
    out.append(("X^(N-1)", [0] * (N - 1) + [-C], None, C))
    return out


@pytest.mark.parametrize("name", ["k_conv-64", "k_conv-4096", "k1_conv-sp", "k_conv_plain-105", "k_conv_plain-1271"])
def test_norm_kernels_on_shaped_polynomials(ring, name):
    """k_norm_twist / k_norm_stage (every radix-2 stage, the max over both outputs of the last) and k_gen_norm (every
    coefficient tile, every evaluation point) on coefficients near Q/4, where the floor is far below the norm: each
    polynomial's largest value sits at its own evaluation point or comes from its own coefficient."""
    ch, O, E = ring(name)
    S, N = ch.ctxt, ch.phim
    Q = ch.product(S)
    C = Q // 4
    cases = peaked(ch, C)
    X = [upload(ch, O, E, f, S) for _, f, _, _ in cases]
    E.profile(True)
    got = E.add_primes_norm(X, S, ch.special)
    E.profile(False)
    assert {conv_kernel(name), norm_kernel(ch)} <= kernels(E), kernels(E)
    fl = ln_floor(N, len(S), Q)
    for (label, f, peak, closed), g in zip(cases, got):
        want = ref_ln(f, ch.m)
        if closed is not None:
            assert abs(want - math.log(closed)) <= 1e-12 * abs(want), (label, want, math.log(closed))
        if peak is not None:
            pts, vals = evaluations(f, ch.m)
            assert vals[pts.index(peak)] >= (1 - 1e-12) * vals.max(), label
        assert_ln(g, want, fl, label)


# ---- d. batch layout

@pytest.mark.parametrize("name,nitems", [("k_conv-64", 65), ("k_conv-64", 130), ("k_conv_plain-105", 65)])
def test_batches_past_one_chunk(ring, name, nitems):
    """65 and 130 items (more than one chunk of 64): item i is c_i X^(k_i) with its own c_i, so each norm must land in its
    own slot: addPrimes, scaleDownToSet (p = 1: delta/P = d_i/P) and breakIntoDigits with its [item*maxdig + i] layout."""
    ch, O, E = ring(name)
    S, Sp, N = ch.ctxt, sorted(ch.ctxt + ch.special), ch.phim
    Q, Pd = ch.product(S), ch.product(ch.special)
    Qd = [ch.product(d) for d in ch.digits]

    def mono(c, k):
        f = [0] * N
        f[k % N] = c
        return f

    # addPrimes
    cs = [(-1) ** i * (Q // 1000) * (i + 1) for i in range(nitems)]
    X = [upload(ch, O, E, mono(c, 7 * i), S) for i, c in enumerate(cs)]
    got = E.add_primes_norm(X, S, ch.special)
    fl = ln_floor(N, len(S), Q)
    for i, c in enumerate(cs):
        assert_ln(got[i], math.log(abs(c)), fl, i)
    assert equal(X[-1], ch, O, mono(cs[-1], 7 * (nitems - 1)), ch.special)
    # scaleDownToSet
    ds = [(-1) ** i * (Pd // 1000) * (i + 1) for i in range(nitems)]
    X = [upload(ch, O, E, [a + Pd * b for a, b in zip(mono(d, 5 * i), mono(i + 1, 5 * i + 1))], Sp) for i, d in enumerate(ds)]
    got = E.scale_down_norm(X, Sp, S, 1)
    for i, d in enumerate(ds):
        assert_norm(got[i], abs(d) / Pd, 4 * len(ch.special) * N * 2.0 ** -64, i)
    assert equal(X[-1], ch, O, mono(nitems, 5 * nitems - 4), S)
    # breakIntoDigits
    es = [[(-1) ** (i + d) * (q // 1000) * (i + 1 + 3 * d) for d, q in enumerate(Qd)] for i in range(nitems)]
    xs = []
    for i, e in enumerate(es):
        x, scale = [0] * N, 1
        for d, (c, q) in enumerate(zip(e, Qd)):
            x = [a + b * scale for a, b in zip(x, mono(c, 3 * i + d))]
            scale *= q
        xs.append(x)
    X = [upload(ch, O, E, x, S) for x in xs]
    D, got = E.break_into_digits_norm(X, S)
    assert got.shape == (nitems, len(ch.digits))
    for i, e in enumerate(es):
        for d, (c, q) in enumerate(zip(e, Qd)):
            assert_ln(got[i, d], math.log(abs(c)), ln_floor(N, len(ch.digits[d]), q), (i, d))
    assert equal(D[-1][1], ch, O, mono(es[-1][1], 3 * (nitems - 1) + 1), Sp)


@pytest.mark.parametrize("name", ["k_conv-64", "k_conv_plain-105"])
def test_digits_norms_across_a_missing_middle_digit(ring, name):
    """breakIntoDigits over digits 0 and 2 only: digit 1 is the zero polynomial the reference carries (norm 0, ln -inf),
    and digit 2's norm lands in its own column, in every item of a batch.  x = d0 + Q0 Q1 d2 mod Q0 Q2: the digit after the
    missing one is still divided by that digit's product."""
    ch, O, E = ring(name)
    rng = np.random.default_rng(4)
    N = ch.phim
    S = ch.digits[0] + ch.digits[2]
    Sp = sorted(S + ch.special)
    Q0, Q1, Q2 = (ch.product(d) for d in ch.digits)
    items = []
    for kind in PATTERNS:
        d0, _ = pattern(kind, Q0, N, 2, rng)
        d2, _ = pattern("scatter" if kind != "scatter" else "table", Q2, N, 2, rng)
        items.append((d0, d2, [po.bal(a + Q0 * Q1 * b, Q0 * Q2) for a, b in zip(d0, d2)]))
    X = [upload(ch, O, E, x, S) for _, _, x in items]
    D, got = E.break_into_digits_norm(X, S)
    assert got.shape == (len(items), 3)
    for it, (d0, d2, x) in enumerate(items):
        ref = digits_of(ch, x, S)
        assert ref[0] == d0 and not any(ref[1]) and ref[2] == d2
        if O is not None:
            rd = O.break_into_digits(rows_of(ch, O, x, S), S)
            assert rd.shape[0] == 3 and all((D[it][d].download(Sp)[Sp] == rd[d][Sp]).all() for d in (0, 2)), it
        assert equal(D[it][2], ch, O, d2, Sp), it
        assert_ln(got[it, 0], ref_ln(d0, ch.m), ln_floor(N, 2, Q0), (it, 0))
        assert got[it, 1] == -math.inf, it
        assert_ln(got[it, 2], ref_ln(d2, ch.m), ln_floor(N, 2, Q2), (it, 2))


# ---- e. hb_bsgs_linear_map_norm

@pytest.mark.parametrize("case", [(0, 3, 5), (1, 3, 5), (1, 2, 18)], ids=["native", "extended", "extended-2-groups"])
def test_bsgs_linear_map_norms(ring, case):
    """The norms of every rotated giant step, item by item: ln ||E_i|| of the digits of x1 and, in the extended form,
    ||delta/P|| of the mod-down of both parts (offsets 8 and 9), against the oracle's rotated giant steps; giant step 0
    has k = 1 and keeps its NaN sentinel, as do the mod-down entries of the native form and the unused digit slots.  18
    giant steps of 2 items are 36 (giant step, item) pairs, more than one group of 32."""
    extended, nitems, ngiant = case
    ch, O, E = ring("k_conv-64", (2, 2))
    X = PowOps(O, ch)
    rng = np.random.default_rng(5 + extended + ngiant)
    S, Sp, N = ch.ctxt, sorted(ch.ctxt + ch.special), ch.phim
    R = Sp if extended else S
    nd, nb, p = len(ch.digits), 2, P_ODD
    Pd = ch.product(ch.special)
    ks = [1] + [units(ch.m, 31)[t % 31] for t in range(ngiant - 1)]

    def rand(idx):
        return O.random(rng, idx)

    b0 = [[rand(R) for _ in range(nb)] for _ in range(nitems)]
    b1 = [[rand(R) for _ in range(nb)] for _ in range(nitems)]
    cs = [[rand(R) for _ in range(nb)] for _ in ks]
    ea = [np.stack([rand(Sp) for _ in range(nd)]) for _ in ks]
    eb = [np.stack([rand(Sp) for _ in range(nd)]) for _ in ks]
    A0 = [E.poly(X.zeros(), Sp) for _ in range(nitems)]
    A1 = [E.poly(X.zeros(), Sp) for _ in range(nitems)]
    E.profile(True)
    got = E.bsgs_linear_map([[E.poly(x, R) for x in it] for it in b0], [[E.poly(x, R) for x in it] for it in b1], S, ks,
                            [[E.poly(x, R) for x in row] for row in cs],
                            [None if k == 1 else [E.poly(a[i], Sp) for i in range(nd)] for a, k in zip(ea, ks)],
                            [None if k == 1 else [E.poly(b[i], Sp) for i in range(nd)] for b, k in zip(eb, ks)],
                            A0, A1, extended=extended, ptxt_space=p, norms=True)
    E.profile(False)
    st = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert "k_norm_stage" in st and st["k_ks_giant"] >= (2 if ngiant * nitems > 32 else 1), st
    assert got.shape == (nitems, ngiant, 10)
    for it in range(nitems):
        r0, r1 = bsgs_reference(X, ch, b0[it], b1[it], cs, ks, None, extended, ea, eb, X.zeros(), X.zeros())
        assert (A0[it].download(Sp)[Sp] == r0[Sp]).all() and (A1[it].download(Sp)[Sp] == r1[Sp]).all(), it
        for t, k in enumerate(ks):
            o = got[it, t]
            if k == 1:
                assert np.isnan(o).all(), (it, t, o)
                continue
            assert np.isnan(o[nd:8]).all(), (it, t, o)
            x0, x1 = X.zeros(), X.zeros()
            for j in range(nb):
                X.muladd(x0, b0[it][j], cs[t][j], R)
                X.muladd(x1, b1[it][j], cs[t][j], R)
            X.automorph(x0, R, k)
            X.automorph(x1, R, k)
            if extended:
                for part, x in ((0, x0), (1, x1)):
                    delta = from_limbs(O.scale_down(x, Sp, S, p, want_delta=True))
                    want = ref_norm_float([float(Fraction(d, Pd)) for d in delta], ch.m)
                    assert_norm(o[8 + part], want, 4 * len(ch.special) * N * 2.0 ** -64, (it, t, part))
            else:
                assert np.isnan(o[8:]).all(), (it, t, o)
            _, polys = O.break_into_digits(x1, S, want_polys=True)
            for i in range(nd):
                dg = from_limbs(polys[i])
                assert_ln(o[i], ref_ln(dg, ch.m), ln_floor(N, len(ch.digits[i]), ch.product(ch.digits[i])), (it, t, i))
