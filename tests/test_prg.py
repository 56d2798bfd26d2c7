"""Device expansion of key-switching rows from a PRG seed (hb_poly_randomize, k_prg_count / k_prg_fill).

NTL::SetSeed(seed) followed by DoubleCRT::randomize() on each poly (src/keys.cpp:1189-1206, src/Ctxt.cpp:191-230,
src/DoubleCRT.cpp:1258-1378), bit for bit against the oracle's restatement of NTL's stream -- which the reference's own
fixture pins (tests/test_oracle.py).  Each parity test runs on the CPU simulator build and, marked gpu, on the H100.
"""
import numpy as np
import pytest

import ntl_prg
import ntl_prg_np as npg
import pyoracle as po
from common import chain
from helib_b200.engine import Engine, HbError
from prg_sim import drop_stale_sim_build

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
SEED256 = 0xB7E151628AED2A6ABF7158809CF4F3C762E7160F38B4DA56A784D9045190CFEF


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def _oracle(primes, phim, idx, seed, npolys):
    st = ntl_prg.set_seed(seed) if isinstance(seed, int) else ntl_prg.RandomStream(ntl_prg.derive_key(bytes(seed).rstrip(b"\0")))
    ch = po.Chain(m=0, p=0, r=1, phim=phim, primes=list(primes))
    return [po.randomize_rows(ch, idx, st.get) for _ in range(npolys)]


def _expand(E, idx, seed, npolys):
    P = [E.poly() for _ in range(npolys)]
    E.randomize(P, idx, seed)
    return [p.download(list(range(E.np))) for p in P]


def _check(E, got, ref, idx):
    for g, r in zip(got, ref):
        for i in range(E.np):
            if i in idx:
                assert [int(v) for v in g[i]] == r[i], f"row {i}"
            else:
                assert not g[i].any(), f"row {i} outside idx was written"


# ---- the vectorised oracle against the scalar restatement (CPU only)

def test_vectorised_stream_matches_scalar_restatement():
    for seed in (0, 1, SEED256, 1 << 700):
        key = npg.seed_key(seed)
        assert key == ntl_prg.derive_key(ntl_prg.zz_bytes(seed))
        ref = b"".join(ntl_prg.chacha20_block(key, i) for i in range(3, 70))
        assert npg.chacha20_blocks(key, 3, 67).tobytes() == ref
    ch, _ = chain(4096, 257, 1, 120, 2)
    for m_, phim, primes in ((4096, ch.phim, ch.primes), (1285, 1024, [257, 3 * 1285 * 4 + 1])):
        idx = list(range(len(primes)))
        st = ntl_prg.set_seed(SEED256)
        bs = npg.BufferStream(SEED256)
        pch = po.Chain(m=m_, p=0, r=1, phim=phim, primes=list(primes))
        for _ in range(2):
            a = po.randomize_rows(pch, idx, st.get)
            b = npg.randomize_rows(primes, phim, idx, bs)
            assert all([int(v) for v in b[i]] == a[i] for i in idx)


# ---- 1. pinned directly by reference output

def test_rows_regenerated_from_reference_matrices(lib):
    """The four matrices of tests/golden/helib_iotest_m12.json (written by a real HElib) store b_i and the 256-bit prgSeed.
    The device expands a_i over ctxt|special from the seed, npolys = n digits in one call; the rows equal the oracle's, and
    b_i + a_i*s - P*prod_{j<i}Q_j*s' leaves one small multiple of p on every prime.  The context is built with m = 8
    (N = 4 = phi(12)): every fixture prime is 1 mod 8, and the expansion only needs the primes and N."""
    from test_oracle import _fixture_chain, _iotest_cases, _regenerate_a
    for case in _iotest_cases():
        ch, roots = _fixture_chain(case)
        assert ch.phim == 4
        m, p = ch.m, ch.p
        E = Engine(8, ch.primes, None, lib=lib)
        rep = po.zms_rep(m)
        pos = {r: j for j, r in enumerate(rep)}
        P = ch.product(ch.special)
        sk = {int(i): row for i, row in case["secret_key"].items()}
        full = sorted(ch.ctxt + ch.special)
        for W in case["ksw"]:
            xpow, spow = W["from"][1], W["from"][0]
            got = _expand(E, full, int(W["prg_seed"]), W["n"])
            ref = _regenerate_a(case, ch, W)
            for d in range(W["n"]):
                for i in full:
                    assert [int(v) for v in got[d][i]] == ref[d][i], (W["from"], d, i)
            for d in range(W["n"]):
                noise = None
                for i, q in enumerate(ch.primes):
                    s_from = [pow(sk[i][pos[rep[j] * xpow % m]], spow, q) for j in range(ch.phim)]
                    fac = P * ch.product([k for j in range(d) for k in ch.digits[j]]) % q
                    rr = [(bb + int(aa) * s - fac * sf) % q for bb, aa, s, sf in zip(W["b"][d][str(i)], got[d][i], sk[i], s_from)]
                    coef = [po.bal(c, q) for c in po.gen_ifft(rr, q, m, roots[i])]
                    assert all(c % p == 0 and abs(c) < 200 * p for c in coef), (W["from"], d, i, coef)
                    assert noise is None or coef == noise
                    noise = coef
                assert any(noise)
        E.close()


# ---- 2. parity where rows span many buffers

SMALL = [(64, 257, 1, 120, 2), (2048, 17, 2, 150, 3), (4096, 257, 1, 60, 2), (8192, -1, 1, 119, 2)]


@pytest.mark.parametrize("cfg", SMALL)
def test_power_of_two_rings_match_oracle(lib, cfg):
    ch, psis = chain(*cfg)
    E = Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=lib)
    allp = list(range(len(ch.primes)))
    for npolys, idx, seed in ((1, allp, SEED256), (3, ch.ctxt + ch.special, 7), (2, allp[::2], b"\x05\x01\x00\x00")):
        got = _expand(E, idx, seed, npolys)
        _check(E, got, _oracle(ch.primes, ch.phim, idx, seed, npolys), idx)


@pytest.mark.parametrize("m,p,bits", [(105, 2, 120), (1285, 2, 120)])
def test_general_m_rings_match_oracle(lib, m, p, bits):
    ch = po.build_mod_chain(m, p, 1, bits, 2)
    E = Engine(m, ch.primes, None, ch.digits, ch.special, lib=lib)
    assert E.N == ch.phim
    idx = ch.ctxt + ch.special
    got = _expand(E, idx, SEED256, 2)
    _check(E, got, _oracle(ch.primes, ch.phim, idx, SEED256, 2), idx)


def test_candidate_widths_one_to_eight_bytes(lib):
    """Primes of 14..60 bits (nb = 2..8, including the fixture's 22-bit width) in one chain, N = 1024, and nb = 1 on a
    small ring."""
    m = 2048
    primes = []
    for bits in (14, 17, 22, 28, 36, 41, 45, 49, 53, 57, 60):
        q = (1 << bits) - m + 1
        while not po.is_prime(q):
            q -= m
        primes.append(q)
    nbs = {((q - 1).bit_length() + 7) // 8 for q in primes}
    assert nbs == set(range(2, 9))
    E = Engine(m, primes, None, lib=lib)
    idx = list(range(len(primes)))
    got = _expand(E, idx, SEED256, 2)
    _check(E, got, _oracle(primes, m // 2, idx, SEED256, 2), idx)
    # nb = 1: a prime below 2^8 needs a small ring
    E1 = Engine(8, [17, 41, 73, 97, 113, 193], None, lib=lib)
    got = _expand(E1, [0, 2, 5], 3, 2)
    _check(E1, got, _oracle([17, 41, 73, 97, 113, 193], 4, [0, 2, 5], 3, 2), [0, 2, 5])


def test_seed_forms(lib):
    """High-order zero bytes do not count, seed 0 is the empty byte string, seeds longer than 64 bytes take a multi-block
    SHA-256 in the key derivation; int and bytes seeds agree."""
    ch, psis = chain(4096, 257, 1, 60, 2)
    E = Engine(ch.m, ch.primes, psis, lib=lib)
    idx = ch.ctxt
    base = _expand(E, idx, SEED256, 1)
    as_bytes = SEED256.to_bytes(32, "little")
    assert all((a == b).all() for a, b in zip(base, _expand(E, idx, as_bytes + b"\0\0\0", 1)))
    zero = _expand(E, idx, 0, 1)
    assert all((a == b).all() for a, b in zip(zero, _expand(E, idx, b"\0\0", 1)))
    _check(E, zero, _oracle(ch.primes, ch.phim, idx, 0, 1), idx)
    long_seed = (1 << 700) + 12345
    _check(E, _expand(E, idx, long_seed, 1), _oracle(ch.primes, ch.phim, idx, long_seed, 1), idx)
    assert not (base[0][idx] == zero[0][idx]).all()


def test_rows_longer_than_the_parallel_window(lib, monkeypatch):
    """HB_PRG_WINDOW caps the buffers k_prg_count scans in parallel; rows that need more finish on the slow path."""
    ch, psis = chain(4096, 257, 1, 120, 2)
    idx = ch.ctxt + ch.special
    ref = _oracle(ch.primes, ch.phim, idx, SEED256, 2)
    for w in ("1", "3", "9"):
        monkeypatch.setenv("HB_PRG_WINDOW", w)
        E = Engine(ch.m, ch.primes, psis, lib=lib)
        _check(E, _expand(E, idx, SEED256, 2), ref, idx)
        E.close()


def test_profile_names_the_two_kernels(lib):
    ch, psis = chain(2048, 17, 2, 150, 3)
    E = Engine(ch.m, ch.primes, psis, lib=lib)
    E.profile(True)
    _expand(E, ch.ctxt, 1, 2)
    E.profile(False)
    prof = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert prof == {"k_prg_count": 2 * len(ch.ctxt), "k_prg_fill": 1}


def test_argument_errors(lib):
    import ctypes as C
    ch, psis = chain(64, 257, 1, 120, 2)
    E = Engine(ch.m, ch.primes, psis, lib=lib)
    P = E.poly()
    for idx in ([1, 0], [0, 0], [0, 2, 2], [0, len(ch.primes)]):
        with pytest.raises(HbError) as ei:
            E.randomize([P], idx, 5)
        assert ei.value.code == HB_ERR_BAD_ARG
    with pytest.raises(HbError) as ei:
        E.randomize([], [0], 5)
    assert ei.value.code == HB_ERR_BAD_ARG
    arr = (C.c_void_p * 1)(P.h)
    idx = (C.c_int32 * 1)(0)
    seed = (C.c_uint8 * 1)(1)
    assert E.lib.hb_poly_randomize(None, 1, idx, 1, seed, 1) == HB_ERR_BAD_ARG
    assert E.lib.hb_poly_randomize(arr, 0, idx, 1, seed, 1) == HB_ERR_BAD_ARG
    assert E.lib.hb_poly_randomize(arr, 1, None, 1, seed, 1) == HB_ERR_BAD_ARG
    assert E.lib.hb_poly_randomize(arr, 1, idx, 1, None, 1) == HB_ERR_BAD_ARG
    assert E.lib.hb_poly_randomize(arr, 1, idx, 1, seed, -1) == HB_ERR_BAD_ARG
    assert E.lib.hb_poly_randomize(arr, 1, idx, 1, None, 0) == 0          # the seed 0
    with pytest.raises(ValueError):
        E.randomize([P], [0], -3)


# ---- 3. full size on the GPU

@pytest.mark.gpu
def test_full_config3_matrix_on_gpu(cuda_lib):
    """All a_i of a config-3 key-switching matrix (BGV m = 2^17, 3 digits over ctxt|special: 3 x 35 rows of 2^16) from one
    seed, bit for bit against the vectorised oracle."""
    from helib_b200 import Chain
    ch = Chain(1 << 17, 257, 1, 1500, 3, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    full = ch.ctxt + ch.special
    n = len(ch.digits)
    assert (n, len(full), E.N) == (3, 35, 1 << 16)
    got = _expand(E, full, SEED256, n)
    bs = npg.BufferStream(SEED256)
    for d in range(n):
        ref = npg.randomize_rows(ch.primes, E.N, full, bs)
        for i in full:
            assert np.array_equal(got[d][i], ref[i]), (d, i)
