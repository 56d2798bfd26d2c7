"""Key-switching matrices held as their PRG seed (hb_poly_create_seeded / hb_poly_expand, seeded evk_a).

HElib keeps a KeySwitch as its b_i rows plus prgSeed and rebuilds every a_i from the seed on each Ctxt::keySwitchDigits
(src/Ctxt.cpp:191-230).  A seeded set keeps the seed and the row schedule of the k_prg_count chain; k_prg_fill regenerates
the rows a call reads.  Checked bit for bit against hb_poly_randomize (itself pinned to the oracle in tests/test_prg.py) and
against the same key switch run with the rows expanded.  Unless marked, each test runs on the CPU simulator build and,
marked gpu, on the H100.
"""
import ctypes as C
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import chain, make, ptxt_space
from helib_b200.engine import Engine, HbError, _arr
from prg_sim import drop_stale_sim_build
from test_cpp_shim import build_exe

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
SEED256 = 0xB7E151628AED2A6ABF7158809CF4F3C762E7160F38B4DA56A784D9045190CFEF


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def _randomized(E, idx, seed, npolys):
    P = [E.poly() for _ in range(npolys)]
    E.randomize(P, idx, seed)
    return [p.download(list(range(E.np))) for p in P]


def _subsets(idx):
    out = [list(idx), idx[:1], idx[-1:], idx[::2]]
    if len(idx) > 2:
        out.append(idx[: len(idx) // 2])      # a level prefix
    return out


def _check_expand(E, idx, seed, npolys):
    """Every subset of rows expanded from the seeded set equals hb_poly_randomize's rows; nothing else is written."""
    ref = _randomized(E, idx, seed, npolys)
    S = E.seeded(npolys, idx, seed)
    for sub in _subsets(idx):
        D = [E.poly() for _ in range(npolys)]
        E.expand(S, D, sub)
        for p in range(npolys):
            got = D[p].download(list(range(E.np)))
            for i in range(E.np):
                if i in sub:
                    assert np.array_equal(got[i], ref[p][i]), (sub, p, i)
                else:
                    assert not got[i].any(), (sub, p, i)


# ---- 1. rows

SMALL = [(64, 257, 1, 120, 2), (2048, 17, 2, 150, 3), (4096, 257, 1, 60, 2), (8192, -1, 1, 119, 2)]


@pytest.mark.parametrize("cfg", SMALL)
def test_power_of_two_rows_equal_randomize(lib, cfg):
    ch, psis = chain(*cfg)
    E = Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=lib)
    allp = list(range(len(ch.primes)))
    for npolys, idx, seed in ((1, allp, SEED256), (3, sorted(ch.ctxt + ch.special), 7), (2, allp[::2], b"\x05\x01\x00\x00")):
        _check_expand(E, idx, seed, npolys)
    E.close()


@pytest.mark.parametrize("m", [105, 1285])
def test_general_m_rows_equal_randomize(lib, m):
    ch = po.build_mod_chain(m, 2, 1, 120, 2)
    E = Engine(m, ch.primes, None, ch.digits, ch.special, lib=lib)
    _check_expand(E, sorted(ch.ctxt + ch.special), SEED256, 2)
    E.close()


def test_candidate_widths_one_to_eight_bytes(lib):
    m = 2048
    primes = []
    for bits in (14, 17, 22, 28, 36, 41, 45, 49, 53, 57, 60):
        q = (1 << bits) - m + 1
        while not po.is_prime(q):
            q -= m
        primes.append(q)
    assert {((q - 1).bit_length() + 7) // 8 for q in primes} == set(range(2, 9))
    E = Engine(m, primes, None, lib=lib)
    _check_expand(E, list(range(len(primes))), SEED256, 2)
    E1 = Engine(8, [17, 41, 73, 97, 113, 193], None, lib=lib)       # nb = 1
    _check_expand(E1, [0, 2, 5], 3, 2)
    E.close(); E1.close()


def test_seed_forms(lib):
    ch, psis = chain(4096, 257, 1, 60, 2)
    E = Engine(ch.m, ch.primes, psis, lib=lib)
    for seed in (SEED256.to_bytes(32, "little") + b"\0\0\0", 0, b"\0\0", (1 << 700) + 12345):
        _check_expand(E, ch.ctxt, seed, 1)
    E.close()


@pytest.mark.parametrize("w", ["1", "2"])
def test_rows_longer_than_the_counting_window(lib, monkeypatch, w):
    """Under HB_PRG_WINDOW every row finishes on k_prg_count's slow path, which records no offsets for its extra buffers:
    creation counts those rows again with their exact need, and the seeded rows still equal hb_poly_randomize's."""
    monkeypatch.setenv("HB_PRG_WINDOW", w)
    ch, psis = chain(4096, 257, 1, 120, 2)
    E = Engine(ch.m, ch.primes, psis, lib=lib)
    _check_expand(E, sorted(ch.ctxt + ch.special), SEED256, 2)
    E.close()


def test_reference_matrices_expanded_from_their_seeds(lib):
    """The four matrices of tests/golden/helib_iotest_m12.json (written by a real HElib): their a_i, expanded from the
    stored prgSeed out of a seeded set, equal the oracle's regeneration."""
    from test_oracle import _fixture_chain, _iotest_cases, _regenerate_a
    for case in _iotest_cases():
        ch, _ = _fixture_chain(case)
        E = Engine(8, ch.primes, None, lib=lib)
        full = sorted(ch.ctxt + ch.special)
        for W in case["ksw"]:
            n = W["n"]
            S = E.seeded(n, full, int(W["prg_seed"]))
            D = [E.poly() for _ in range(n)]
            E.expand(S, D, full)
            ref = _regenerate_a(case, ch, W)
            for d in range(n):
                got = D[d].download(full)
                for i in full:
                    assert [int(v) for v in got[i]] == ref[d][i], (W["from"], d, i)
        E.close()


# ---- 2. key switches: seeded evk_a against the same a_i expanded

def _keys(E, ch, rng, seed):
    """A matrix over ctxt|special: seeded a_i, the same a_i expanded, random b_i."""
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    SA = E.seeded(nd, full, seed)
    EA = [E.poly() for _ in range(nd)]
    E.randomize(EA, full, seed)
    EB = [E.poly(_rand(ch, rng, full, E.N), full) for _ in range(nd)]
    return SA, EA, EB


def _rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def _same(E, A, B, idx):
    return all(np.array_equal(a.download(idx)[idx], b.download(idx)[idx]) for a, b in zip(A, B))


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (4096, 257, 1, 60, 2)])
def test_keyswitch_digits(lib, cfg):
    ch, psis, O, E = make(lib, *cfg)
    rng = np.random.default_rng(11)
    SA, EA, EB = _keys(E, ch, rng, SEED256)
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    c2 = E.poly(_rand(ch, rng, S, E.N), S)
    digs = E.break_into_digits([c2], S)
    outs = []
    for A in (EA, SA):
        X0, X1 = E.poly(_rand(ch, np.random.default_rng(1), Sp, E.N), Sp), E.poly()
        E.keyswitch_digits(digs, Sp, A[: len(digs[0])], EB[: len(digs[0])], [X0], [X1])
        outs.append((X0, X1))
    assert _same(E, outs[0], outs[1], Sp)
    E.close()


@pytest.mark.parametrize("cfg", [(4096, 17, 1, 160, 3), (1 << 17, 257, 1, 230, 2)])
def test_keyswitch_digits_fused_with_own_rows_and_an_owned_subset(lib, cfg):
    """scal and own/own_dig as Ctxt::keySwitchPart uses them, on every row of S|special and on half of them (the rows one
    rank of the prime-sharded key switch owns)."""
    ch, psis, O, E = make(lib, *cfg, nthreads=8)
    rng = np.random.default_rng(41)
    SA, EA, EB = _keys(E, ch, rng, 12345)
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    nd = len(ch.digits)
    D = [E.poly(_rand(ch, rng, Sp, E.N), Sp) for _ in range(nd)]
    OWN = E.poly(_rand(ch, rng, S, E.N), S)
    P = 1
    for i in ch.special:
        P *= ch.primes[i]
    init = [_rand(ch, rng, Sp, E.N) for _ in range(2)]
    for rows in (Sp, Sp[::2]):
        scal = [P % ch.primes[r] if r in S else 0 for r in rows]
        own_dig = [next(d for d in range(nd) if r in ch.digits[d]) if r in S else -1 for r in rows]
        outs = []
        for A in (EA, SA):
            C0, C1 = E.poly(init[0], Sp), E.poly(init[1], Sp)
            E.keyswitch_digits_fused([D], rows, A, EB, [C0], [C1], scal, own=[OWN], own_dig=own_dig)
            outs.append((C0, C1))
        assert _same(E, outs[0], outs[1], Sp), len(rows)
    E.close()


def _relin(E, ch, S, A, B, cs):
    C0, C1, C2 = ([E.poly(c[k], S) for c in cs] for k in range(3))
    E.relinearize(C0, C1, C2, S, A, B)
    return C0 + C1


def test_relinearize_fused_and_step_by_step(lib):
    """N = 2^16 takes the fused relinearisation (regeneration once, before its item chunks); an index set with a digit
    hole takes the step-by-step path."""
    ch, psis, O, E = make(lib, 1 << 17, 257, 1, 230, 3, nthreads=8)
    rng = np.random.default_rng(77)
    SA, EA, EB = _keys(E, ch, rng, SEED256)
    hole = [i for i in ch.ctxt if i not in ch.digits[0]]
    assert hole and len(hole) < len(ch.ctxt)
    for S in (ch.ctxt, ch.ctxt[:-1], hole):
        Sp = sorted(S + ch.special)
        cs = [[_rand(ch, rng, S, E.N) for _ in range(3)] for _ in range(2)]
        assert _same(E, _relin(E, ch, S, EA, EB, cs), _relin(E, ch, S, SA, EB, cs), Sp), len(S)
    E.close()


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (8192, -1, 1, 119, 2)])
def test_mul_relin_moddown_at_a_lower_level(lib, cfg):
    ch, psis, O, E = make(lib, *cfg)
    p = ptxt_space(ch)
    rng = np.random.default_rng(6)
    SA, EA, EB = _keys(E, ch, rng, 99)
    S_in, S = ch.ctxt, ch.ctxt[:-1]
    ops = [[_rand(ch, rng, S_in, E.N) for _ in range(4)] for _ in range(2)]
    outs = []
    for A in (EA, SA):
        A0, A1, B0, B1 = ([E.poly(o[k], S_in) for o in ops] for k in range(4))
        E.mul_relin_moddown(A0, A1, B0, B1, S_in, S, p, A, EB)
        outs.append(A0 + A1)
    assert _same(E, outs[0], outs[1], S)
    E.close()


def _hoisted(E, ch, rng, m, ks):
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    c0, c1 = _rand(ch, rng, S, E.N), _rand(ch, rng, S, E.N)
    C0 = E.poly(c0, S)
    digs = E.break_into_digits([E.poly(c1, S)], S)
    for j, k in enumerate(ks):
        SA, EA, EB = _keys(E, ch, rng, 1000 + j)       # every amount has its own matrix
        outs = []
        for A in (EA, SA):
            O0, O1 = E.poly(), E.poly()
            E.automorph_keyswitch_digits(digs, S, [C0], k, A, EB, [O0], [O1])
            outs.append((O0, O1))
        assert _same(E, outs[0], outs[1], Sp), k


@pytest.mark.parametrize("cfg", [(64, 257, 1, 120, 2), (8192, -1, 1, 119, 2)])
def test_hoisted_rotation_power_of_two(lib, cfg):
    ch, psis, O, E = make(lib, *cfg)
    _hoisted(E, ch, np.random.default_rng(31), ch.m, (3, 5, ch.m - 1))
    E.close()


@pytest.mark.parametrize("m", [105, 1285])
def test_hoisted_rotation_general_m(lib, m):
    ch = po.build_mod_chain(m, 2, 1, 120, 2)
    E = Engine(m, ch.primes, None, ch.digits, ch.special, lib=lib)
    ks = [t for t in range(2, m) if np.gcd(t, m) == 1][:2] + [m - 1]
    _hoisted(E, ch, np.random.default_rng(32), m, ks)
    E.close()


# ---- 3. rejection (simulator)

def _sim_engine(sim_lib):
    ch, psis = chain(4096, 257, 1, 60, 2)
    return ch, Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=sim_lib)


def _calls(E, ch, X):
    """Every entry point with the seeded poly X in one position that is not evk_a, as (name, thunk) pairs."""
    L = E.lib
    S, full = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    P = lambda: E.poly()                                            # noqa: E731
    u64 = C.POINTER(C.c_uint64)
    i32 = C.POINTER(C.c_int32)
    idx = np.array(S, dtype=np.int32)
    ip = idx.ctypes.data_as(i32)
    host = np.zeros((E.np, E.N), dtype=np.uint64)
    hp = host.ctypes.data_as(u64)
    big = np.zeros(E.N * 8 * (E.np + 1), dtype=np.uint64)
    bp = big.ctypes.data_as(u64)
    i64 = np.zeros(E.N * 4, dtype=np.int64).ctypes.data_as(C.POINTER(C.c_int64))
    dbl = np.zeros(64, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))
    sc = np.ones(E.np, dtype=np.uint64)
    scp = sc.ctypes.data_as(u64)
    own_dig = np.full(len(full), -1, dtype=np.int32)
    ndo = C.c_int()
    nbytes = C.c_uint64()
    seed = (C.c_uint8 * 1)(5)
    hbuf = C.create_string_buffer(64)
    sbuf = C.create_string_buffer(1 << 16)
    A = lambda *polys: _arr(_keep(list(polys)))                    # noqa: E731
    EA = E.seeded(nd, full, 3)
    EB = [P() for _ in range(nd)]
    pos = lambda k, n=1: [X if i == k else P() for i in range(n)]  # noqa: E731
    calls = [
        ("upload", lambda: L.hb_poly_upload(X.h, ip, len(idx), hp)),
        ("download", lambda: L.hb_poly_download(X.h, ip, len(idx), hp)),
        ("download_async", lambda: L.hb_poly_download_async(X.h, ip, len(idx), hp)),
        ("serialized_size", lambda: L.hb_poly_serialized_size(X.h, 1, C.byref(nbytes))),
        ("serialize", lambda: L.hb_poly_serialize(X.h, ip, 1, sbuf, C.c_uint64(len(sbuf)))),
        ("deserialize", lambda: L.hb_poly_deserialize(X.h, sbuf, C.c_uint64(len(sbuf)), ip, C.byref(ndo))),
        ("randomize", lambda: L.hb_poly_randomize(A(X), 1, ip, len(idx), seed, 1)),
        ("expand(dst)", lambda: L.hb_poly_expand(A(EA[0]), A(X), 1, ip, len(idx))),
        ("ipc_export", lambda: L.hb_poly_ipc_export(X.h, hbuf)),
        ("ntt_fwd", lambda: L.hb_ntt_fwd(A(X), 1, ip, len(idx))),
        ("ntt_inv", lambda: L.hb_ntt_inv(A(X), 1, ip, len(idx))),
        ("scale_rows", lambda: L.hb_scale_rows(A(X), 1, ip, len(idx), scp)),
        ("scale_by_primes", lambda: L.hb_scale_by_primes(A(X), 1, ip, 1, ip, 1, 0)),
        ("zero_rows", lambda: L.hb_zero_rows(A(X), 1, ip, len(idx))),
        ("add_primes_and_scale", lambda: L.hb_add_primes_and_scale(A(X), 1, ip, len(idx), _ia(ch.special), len(ch.special))),
        ("add_primes", lambda: L.hb_add_primes(A(X), 1, ip, len(idx), _ia(ch.special), len(ch.special))),
        ("add_primes_norm", lambda: L.hb_add_primes_norm(A(X), 1, ip, len(idx), _ia(ch.special), len(ch.special), dbl)),
        ("scale_down", lambda: L.hb_scale_down(A(X), 1, _ia(full), len(full), ip, len(idx), C.c_uint64(1))),
        ("scale_down_norm", lambda: L.hb_scale_down_norm(A(X), 1, _ia(full), len(full), ip, len(idx), C.c_uint64(1), dbl)),
        ("to_poly", lambda: L.hb_to_poly(X.h, ip, len(idx), 0, bp, len(idx) + 1)),
        ("to_poly_mod_p", lambda: L.hb_to_poly_mod_p(X.h, ip, len(idx), C.c_uint64(257), C.c_uint64(1), i64)),
        ("dcrt_to_powerful", lambda: L.hb_dcrt_to_powerful(X.h, ip, len(idx), bp, len(idx) + 1)),
        ("raw_mod_switch", lambda: L.hb_raw_mod_switch(X.h, ip, len(idx), C.c_uint64(257), C.c_uint64(257), i64)),
        ("from_i64", lambda: L.hb_poly_from_i64(A(X), 1, ip, len(idx), i64)),
        ("from_limbs", lambda: L.hb_poly_from_limbs(A(X), 1, ip, len(idx), bp, 1)),
        ("conv_make_y(src)", lambda: L.hb_conv_make_y(A(X), 1, ip, len(idx), ip, 1, A(P()))),
        ("conv_make_y(y)", lambda: L.hb_conv_make_y(A(P()), 1, ip, len(idx), ip, 1, A(X))),
        ("conv_make_y_bcast(peer)", lambda: L.hb_conv_make_y_bcast(A(P()), 1, ip, len(idx), ip, 1, A(P()), A(X), 1)),
        ("conv_from_y(y)", lambda: L.hb_conv_from_y(A(X), 1, ip, len(idx), _ia(ch.special), len(ch.special), C.c_uint64(1), A(P()), 0)),
        ("conv_from_y(dst)", lambda: L.hb_conv_from_y(A(P()), 1, ip, len(idx), _ia(ch.special), len(ch.special), C.c_uint64(1), A(X), 0)),
        ("tensor(o2)", lambda: L.hb_tensor(A(P()), A(P()), A(P()), A(P()), A(P()), A(P()), A(X), 1, ip, len(idx))),
        ("automorph(dst)", lambda: L.hb_automorph(A(X), A(P()), 1, ip, len(idx), C.c_uint64(3))),
        ("automorph(src)", lambda: L.hb_automorph(A(P()), A(X), 1, ip, len(idx), C.c_uint64(3))),
        ("sub_div_by_primes", lambda: L.hb_sub_div_by_primes(A(P()), A(X), 1, ip, 1, ip, 1)),
    ]
    for k in range(2):
        calls.append((f"pointwise[{k}]", lambda k=k: L.hb_pointwise(2, A(*pos(k, 2)[:1]), A(*pos(k, 2)[1:]), 1, ip, len(idx))))
    for k in range(3):
        calls.append((f"muladd[{k}]", lambda k=k: L.hb_muladd(*[A(p) for p in pos(k, 3)], 1, ip, len(idx))))
    for k in range(6):
        calls.append((f"tensor[{k}]", lambda k=k: L.hb_tensor(*[A(p) for p in pos(k, 7)], 1, ip, len(idx))))
    calls.append(("break_into_digits(src)", lambda: L.hb_break_into_digits(A(X), 1, ip, len(idx), A(*[P() for _ in range(nd)]), nd, C.byref(ndo))))
    calls.append(("break_into_digits(digit)", lambda: L.hb_break_into_digits(A(P()), 1, ip, len(idx), A(*pos(nd - 1, nd)), nd, C.byref(ndo))))
    calls.append(("break_into_digits_norm", lambda: L.hb_break_into_digits_norm(A(P()), 1, ip, len(idx), A(*pos(0, nd)), nd, C.byref(ndo), dbl)))
    fp, nf = _ia(full), len(full)
    fsc = np.ones(nf, dtype=np.uint64).ctypes.data_as(u64)
    odp = own_dig.ctypes.data_as(i32)
    # key switches: digits, evk_b, outputs, own, c0 (evk_a is the seeded EA throughout)
    for k in range(nd):
        calls.append((f"keyswitch_digits(digit {k})", lambda k=k: L.hb_keyswitch_digits(A(*pos(k, nd)), nd, nd, 1, fp, nf, A(*EA), A(*EB), A(P()), A(P()))))
        calls.append((f"keyswitch_digits(evk_b {k})", lambda k=k: L.hb_keyswitch_digits(A(*[P() for _ in range(nd)]), nd, nd, 1, fp, nf, A(*EA), A(*pos(k, nd)), A(P()), A(P()))))
        calls.append((f"automorph_keyswitch(digit {k})", lambda k=k: L.hb_automorph_keyswitch_digits(A(*pos(k, nd)), nd, nd, 1, ip, len(idx), A(P()), C.c_uint64(3), A(*EA), A(*EB), A(P()), A(P()))))
        calls.append((f"automorph_keyswitch(evk_b {k})", lambda k=k: L.hb_automorph_keyswitch_digits(A(*[P() for _ in range(nd)]), nd, nd, 1, ip, len(idx), A(P()), C.c_uint64(3), A(*EA), A(*pos(k, nd)), A(P()), A(P()))))
        calls.append((f"relinearize(evk_b {k})", lambda k=k: L.hb_relinearize(A(P()), A(P()), A(P()), 1, ip, len(idx), A(*EA), A(*pos(k, nd)), nd)))
        calls.append((f"mul_relin_moddown(evk_b {k})", lambda k=k: L.hb_mul_relin_moddown(A(P()), A(P()), A(P()), A(P()), 1, ip, len(idx), ip, len(idx), C.c_uint64(257), A(*EA), A(*pos(k, nd)), nd)))
        calls.append((f"keyswitch_digits_fused(evk_b {k})", lambda k=k: L.hb_keyswitch_digits_fused(A(*[P() for _ in range(nd)]), nd, nd, 1, fp, nf, A(*EA), A(*pos(k, nd)), A(P()), A(P()), fsc, A(P()), odp)))
    for k in range(2):
        calls.append((f"keyswitch_digits(out{k})", lambda k=k: L.hb_keyswitch_digits(A(*[P() for _ in range(nd)]), nd, nd, 1, fp, nf, A(*EA), A(*EB), *[A(p) for p in pos(k, 2)])))
        calls.append((f"keyswitch_digits_fused(out{k})", lambda k=k: L.hb_keyswitch_digits_fused(A(*[P() for _ in range(nd)]), nd, nd, 1, fp, nf, A(*EA), A(*EB), *[A(p) for p in pos(k, 2)], fsc, A(P()), odp)))
        calls.append((f"automorph_keyswitch(out{k})", lambda k=k: L.hb_automorph_keyswitch_digits(A(*[P() for _ in range(nd)]), nd, nd, 1, ip, len(idx), A(P()), C.c_uint64(3), A(*EA), A(*EB), *[A(p) for p in pos(k, 2)])))
    calls.append(("keyswitch_digits_fused(own)", lambda: L.hb_keyswitch_digits_fused(A(*[P() for _ in range(nd)]), nd, nd, 1, fp, nf, A(*EA), A(*EB), A(P()), A(P()), fsc, A(X), odp)))
    calls.append(("keyswitch_digits_fused(digit)", lambda: L.hb_keyswitch_digits_fused(A(*pos(0, nd)), nd, nd, 1, fp, nf, A(*EA), A(*EB), A(P()), A(P()), fsc, A(P()), odp)))
    calls.append(("automorph_keyswitch(c0)", lambda: L.hb_automorph_keyswitch_digits(A(*[P() for _ in range(nd)]), nd, nd, 1, ip, len(idx), A(X), C.c_uint64(3), A(*EA), A(*EB), A(P()), A(P()))))
    for k in range(3):
        calls.append((f"relinearize(c{k})", lambda k=k: L.hb_relinearize(*[A(p) for p in pos(k, 3)], 1, ip, len(idx), A(*EA), A(*EB), nd)))
    for k in range(4):
        calls.append((f"mul_relin_moddown[{k}]", lambda k=k: L.hb_mul_relin_moddown(*[A(p) for p in pos(k, 4)], 1, ip, len(idx), ip, len(idx), C.c_uint64(257), A(*EA), A(*EB), nd)))
    return calls


_KEEP = []


def _keep(x):
    """The handles of a call's temporary polys must outlive the call."""
    _KEEP.append(x)
    return x


def _ia(lst):
    a = np.ascontiguousarray(np.array(lst, dtype=np.int32))
    _KEEP.append(a)
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def test_a_seeded_poly_is_rejected_everywhere_but_evk_a(sim_lib):
    ch, E = _sim_engine(sim_lib)
    X = E.seeded(1, ch.ctxt, 5)[0]
    calls = _calls(E, ch, X)
    assert len(calls) > 60
    for name, f in calls:
        E.sync()
        before = E.stats()["launches"]
        rc = f()
        assert rc == HB_ERR_BAD_ARG, (name, rc, E.lib.hb_last_error())
        assert E.stats()["launches"] == before, name
    E.close()


def test_rows_outside_the_seeded_set(sim_lib):
    ch, E = _sim_engine(sim_lib)
    rng = np.random.default_rng(2)
    nd = len(ch.digits)
    lower = sorted(ch.ctxt[:-1] + ch.special)
    SA = E.seeded(nd, lower, 3)                   # a matrix that lacks the top ctxt prime
    EB = [E.poly(_rand(ch, rng, sorted(ch.ctxt + ch.special), E.N), sorted(ch.ctxt + ch.special)) for _ in range(nd)]
    with pytest.raises(HbError) as ei:
        E.expand(SA, [E.poly() for _ in range(nd)], [ch.ctxt[-1]])
    assert ei.value.code == HB_ERR_INDEX_SET
    E.reset_stats()
    S = ch.ctxt
    cs = [[_rand(ch, rng, S, E.N) for _ in range(3)]]
    C0, C1, C2 = ([E.poly(c[k], S) for c in cs] for k in range(3))
    E.sync(); E.reset_stats()
    with pytest.raises(HbError) as ei:
        E.relinearize(C0, C1, C2, S, SA, EB)
    assert ei.value.code == HB_ERR_INDEX_SET
    assert E.stats()["launches"] == 0
    # one level lower the same matrix covers every row the call reads
    E.relinearize(C0, C1, C2, ch.ctxt[:-1], SA, EB)
    E.close()


def test_argument_errors_match_randomize(sim_lib):
    ch, E = _sim_engine(sim_lib)
    for idx in ([1, 0], [0, 0], [0, 2, 2], [0, len(ch.primes)]):
        with pytest.raises(HbError) as ei:
            E.seeded(1, idx, 5)
        assert ei.value.code == HB_ERR_BAD_ARG
    with pytest.raises(HbError) as ei:
        E.seeded(0, [0], 5)
    assert ei.value.code == HB_ERR_BAD_ARG
    out = (C.c_void_p * 1)()
    idx = (C.c_int32 * 1)(0)
    seed = (C.c_uint8 * 1)(1)
    L = E.lib
    assert L.hb_poly_create_seeded(None, 1, idx, 1, seed, 1, out) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, 1, idx, 1, seed, 1, None) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, -1, idx, 1, seed, 1, out) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, 1, None, 1, seed, 1, out) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, 1, idx, 1, None, 1, out) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, 1, idx, 1, seed, -1, out) == HB_ERR_BAD_ARG
    assert L.hb_poly_create_seeded(E.h, 1, idx, 1, None, 0, out) == 0      # the seed 0
    L.hb_poly_destroy(out[0])
    # expand: `seeded` must hold seeded polys
    P = E.poly()
    with pytest.raises(HbError) as ei:
        E.expand([P], [E.poly()], [0])
    assert ei.value.code == HB_ERR_BAD_ARG
    E.close()


# ---- 4. memory (simulator)

def test_device_memory_of_seeded_matrices(sim_lib):
    ch, psis = chain(4096, 257, 1, 120, 2)
    E = Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=sim_lib)
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    dense = len(ch.primes) * E.N * 8
    E.seeded(nd, full, 1)                                # context scratch of the count chain, then the handles go
    base = E.stats()["device_bytes"]
    one = E.seeded(nd, full, 2)
    sched = E.stats()["device_bytes"] - base
    assert 0 < sched < dense // 4, (sched, dense)
    K = 5
    more = [E.seeded(nd, full, 10 + j) for j in range(K - 1)]
    assert E.stats()["device_bytes"] - base <= K * sched
    del more
    assert E.stats()["device_bytes"] == base + sched
    # the first seeded key switch adds the key scratch once (nd full-height polys, apart from the digit pool, which an
    # expanded-key call has already sized); the second adds nothing, and the bits are those of the expanded key
    rng = np.random.default_rng(4)
    EA = [E.poly() for _ in range(nd)]
    E.randomize(EA, full, 2)
    EB = [E.poly(_rand(ch, rng, full, E.N), full) for _ in range(nd)]
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    cs = [[_rand(ch, rng, S, E.N) for _ in range(3)] for _ in range(2)]
    ref = [x.download(Sp) for x in _relin(E, ch, S, EA, EB, cs)]
    warm = E.stats()["device_bytes"]
    outs = [_relin(E, ch, S, one, EB, cs) for _ in range(2)]
    del outs
    assert E.stats()["device_bytes"] == warm + nd * dense
    got = [x.download(Sp) for x in _relin(E, ch, S, one, EB, cs)]
    assert all(np.array_equal(a[Sp], b[Sp]) for a, b in zip(ref, got))
    assert E.stats()["device_bytes"] == warm + nd * dense
    del one
    assert E.stats()["device_bytes"] == warm + nd * dense - sched
    E.close()


# ---- 6. the C++ mirror (tests/cpp/test_seeded_keys.cpp): KeySwitch::compress, readFrom(..., false), copies, hoisting

CPP_SEED = "7f3c19a2d05be8416c2e9db3f70815aa4c6e21d8930b5f7ee2a1c4d6089b3e51"


def test_mirror_with_compressed_matrices_on_simulator():
    r = subprocess.run([build_exe("test_seeded_keys", sim=True), CPP_SEED], capture_output=True, text=True)
    assert r.returncode == 0 and "seeded keys OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_with_compressed_matrices_on_gpu():
    r = subprocess.run([build_exe("test_seeded_keys"), CPP_SEED], capture_output=True, text=True)
    assert r.returncode == 0 and "seeded keys OK" in r.stdout, r.stdout + r.stderr


# ---- 5. full size on the GPU

@pytest.mark.gpu
def test_full_config3_relinearize_seeded_and_in_a_cuda_graph(cuda_lib):
    """A config-3 relinearisation (BGV m = 2^17, 26 ctxt + 9 special primes, 3 digits, 8 items) with a seeded matrix gives
    the bits of the expanded one; the same step captured into a CUDA graph and replayed twice gives them again."""
    import torch
    from helib_b200 import Chain
    ch = Chain(1 << 17, 257, 1, 1500, 3, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    rng = np.random.default_rng(3)
    SA = E.seeded(nd, full, SEED256)
    EA = [E.poly() for _ in range(nd)]
    E.randomize(EA, full, SEED256)
    EB = [E.poly(_rand(ch, rng, full, E.N), full) for _ in range(nd)]
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    B = 8
    cs = [[_rand(ch, rng, S, E.N) for _ in range(3)] for _ in range(B)]
    ref = [x.download(Sp) for x in _relin(E, ch, S, EA, EB, cs)]
    got = [x.download(Sp) for x in _relin(E, ch, S, SA, EB, cs)]
    assert all(np.array_equal(a[Sp], b[Sp]) for a, b in zip(ref, got))
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    E.set_stream(side.cuda_stream)
    C0, C1, C2 = ([E.poly() for _ in range(B)] for _ in range(3))
    K0, K1, K2 = ([E.poly(c[k], S) for c in cs] for k in range(3))

    def step():
        E.pointwise("copy", C0 + C1 + C2, K0 + K1 + K2, S)
        E.relinearize(C0, C1, C2, S, SA, EB)

    step()                                                 # warm: digit pool and key scratch exist before the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        step()
    for _ in range(2):
        for x in C0 + C1:
            x.upload(np.zeros((E.np, E.N), dtype=np.uint64), Sp)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert all(np.array_equal(a[Sp], x.download(Sp)[Sp]) for a, x in zip(ref, C0 + C1))
    torch.cuda.set_stream(torch.cuda.default_stream())
    E.close()
