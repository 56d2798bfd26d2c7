"""Squaring on the device: hb_square_tensor (k1_fwd_blk_square) and hb_square_relin_moddown.

Ctxt::square is multiplyBy(*this); multLowLvl's squaring branch brings the one ciphertext to its natural prime set and forms
tensorProduct(*this, *this) (src/Ctxt.cpp:1704-1708).  hb_square_tensor must equal the oracle's scale-down of both parts
followed by the tensor of (x, x), on the register path (k1_fwd_blk_square) and on the generic one (general m, small N,
HB_FORCE_V0, nothing dropped), and its norms must be the doubles hb_scale_down_norm returns; hb_square_relin_moddown must
equal the oracle's square + relinearise + mod-down and, bit for bit, hb_mul_relin_moddown on (x, copy of x).  Every body
runs on the CPU simulator build and, marked gpu, on the H100; the code generation of the kernel is checked on sm_90a
without a GPU."""
import gc
import os
import re
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import make, ptxt_space, rows_equal
from helib_b200.engine import Engine, HbError
from test_codegen import CSRC, _depots, _frames, _nvcc
from test_engine_parity import oracle_mul_relin_moddown
from test_value_ranges import operand, top_chain, top_keys

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
SEED = 0x452821E638D01377BE5466CF34E90C6C


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


@pytest.fixture
def closing():
    """closing(E) -> E: the engine is closed after the test, once the test's polys are gone.  Engine.close is what frees a
    context's scratch (conversion tables, transform scratch, digit and s^2 pools); without it every full-size ring a test
    builds would stay on the device for the rest of the session."""
    made = []
    yield lambda E: made.append(E) or E
    gc.collect()
    for E in made:
        E.close()


def kernels(E):
    return {r["kernel"]: r["launches"] for r in E.profile_results()}


def rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def keys(E, ch, rng, seeded):
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    if seeded:
        SA = E.seeded(nd, full, SEED)
        EA = [E.poly() for _ in range(nd)]
        E.randomize(EA, full, SEED)
    else:
        EA = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
        SA = EA
    EB = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    ea = np.stack([p.download(full) for p in EA])
    eb = np.stack([p.download(full) for p in EB])
    return SA, EA, EB, ea, eb


def oracle_square_tensor(O, ch, x0, x1, S_in, S, p):
    """bringToSet(S) of both parts, then tensorProduct(x, x)."""
    a0, a1 = x0.copy(), x1.copy()
    O.scale_down(a0, S_in, S, p)
    O.scale_down(a1, S_in, S, p)
    return O.tensor(a0, a1, a0, a1, S)


def copies(E, P, idx):
    return [E.poly(x.download(idx), idx) for x in P]


# ---- 1. hb_square_tensor against the oracle, and its norms against hb_scale_down_norm

@pytest.mark.parametrize("m, p, S_in_kind, ndrop, nitems", [
    (8192, 257, "ctxt", 1, 3),
    (8192, 2, "ctxt", 2, 2),
    (8192, 1, "ctxt", 1, 1),
    (8192, 257, "ctxt+special", 1, 2),   # the special primes dropped together with a ctxt prime
    (8192, 257, "ctxt", 0, 2),           # nothing dropped: k1_tensor
    (1 << 17, 1, "ctxt", 1, 2),          # N = 2^16
], ids=["p257-drop1", "p2-drop2", "p1-drop1", "p257-special", "p257-nodrop", "n65536-p1"])
def test_square_tensor_matches_oracle_and_norms(closing, lib, m, p, S_in_kind, ndrop, nitems):
    ch, psis, O, E = make(lib, m, -1 if p == 1 else 257, 1, 240 if ndrop > 1 else 119, 2)
    closing(E)
    rng = np.random.default_rng(301)
    S_in = sorted(ch.ctxt + ch.special) if S_in_kind == "ctxt+special" else ch.ctxt
    S = ch.ctxt[:len(ch.ctxt) - ndrop]
    xs = [(rand(ch, rng, S_in, E.N), rand(ch, rng, S_in, E.N)) for _ in range(nitems)]
    A0, A1 = [E.poly(x[0], S_in) for x in xs], [E.poly(x[1], S_in) for x in xs]
    ref = [copies(E, [A0[i], A1[i]], S_in) for i in range(nitems)]
    O2 = [E.poly() for _ in range(nitems)]
    E.profile(True)
    norms = E.square_tensor(A0, A1, O2, S_in, S, p, norms=True)
    E.profile(False)
    ran = kernels(E)
    for i, (x0, x1) in enumerate(xs):
        t = oracle_square_tensor(O, ch, x0, x1, S_in, S, p)
        for k, P in enumerate((A0[i], A1[i], O2[i])):
            assert rows_equal(P.download(S), t[k], S), (i, k)
    want = E.scale_down_norm([x for r in ref for x in r], S_in, S, p)
    assert np.array_equal(norms.reshape(-1), want), (norms, want)
    if ndrop == 0:
        assert "k1_tensor" in ran and "k1_fwd_blk_square" not in ran and not norms.any(), ran
    else:
        assert ran.get("k1_fwd_blk_square") and "k1_tensor" not in ran and "k1_fwd_blk_subscale" not in ran, ran


@pytest.mark.parametrize("case", ["general-m", "small-n", "force-v0"])
def test_square_tensor_generic_path(closing, lib, monkeypatch, case):
    """General m (Bluestein rows), N not a multiple of 512 and HB_FORCE_V0: the scale-down and the in-place k_pw_tensor,
    against the oracle (power-of-two m) or the composition of hb_scale_down and hb_tensor on copies (general m)."""
    if case == "force-v0":
        monkeypatch.setenv("HB_FORCE_V0", "1")
    if case == "general-m":
        ch = po.build_mod_chain(45, 2, 1, 120, 2)
        O, E = None, Engine(45, ch.primes, None, ch.digits, ch.special, lib=lib)
        closing(E)
    else:
        ch, psis, O, E = make(lib, 256 if case == "small-n" else 8192, 257, 1, 119, 2)
        closing(E)
    p = ptxt_space(ch)
    rng = np.random.default_rng(302)
    S_in, S = ch.ctxt, ch.ctxt[:-1]
    xs = [(rand(ch, rng, S_in, E.N), rand(ch, rng, S_in, E.N)) for _ in range(2)]
    A0, A1 = [E.poly(x[0], S_in) for x in xs], [E.poly(x[1], S_in) for x in xs]
    C0, C1 = [copies(E, [a], S_in)[0] for a in A0], [copies(E, [a], S_in)[0] for a in A1]
    O2 = [E.poly() for _ in range(2)]
    E.profile(True)
    norms = E.square_tensor(A0, A1, O2, S_in, S, p, norms=True)
    E.profile(False)
    ran = kernels(E)
    assert "k1_fwd_blk_square" not in ran and "k_pw_tensor" in ran, ran
    want = E.scale_down_norm([x for i in range(2) for x in (C0[i], C1[i])], S_in, S, p)
    assert np.array_equal(norms.reshape(-1), want)
    T = [[E.poly() for _ in range(2)] for _ in range(3)]
    E.tensor(C0, C1, C0, C1, *T, S)
    for i in range(2):
        for k, P in enumerate((A0[i], A1[i], O2[i])):
            assert rows_equal(P.download(S), T[k][i].download(S), S), (i, k)
        if O is not None:
            t = oracle_square_tensor(O, ch, *xs[i], S_in, S, p)
            for k, P in enumerate((A0[i], A1[i], O2[i])):
                assert rows_equal(P.download(S), t[k], S), (i, k)


# ---- 2. hb_square_relin_moddown against the oracle and hb_mul_relin_moddown(x, copy of x)

def square_case(E, ch, O, S_in, S, p, nitems, seeded, rng_seed=303):
    rng = np.random.default_rng(rng_seed)
    SA, EA, EB, ea, eb = keys(E, ch, rng, seeded)
    xs = [(rand(ch, rng, S_in, E.N), rand(ch, rng, S_in, E.N)) for _ in range(nitems)]
    A0, A1 = [E.poly(x[0], S_in) for x in xs], [E.poly(x[1], S_in) for x in xs]
    M0, M1 = copies(E, A0, S_in), copies(E, A1, S_in)
    B0, B1 = copies(E, A0, S_in), copies(E, A1, S_in)
    E.mul_relin_moddown(M0, M1, B0, B1, S_in, S, p, EA, EB)
    E.profile(True)
    E.square_relin_moddown(A0, A1, S_in, S, p, SA, EB)
    E.profile(False)
    ran = kernels(E)
    for i in range(nitems):
        assert rows_equal(A0[i].download(S), M0[i].download(S), S), i
        assert rows_equal(A1[i].download(S), M1[i].download(S), S), i
        if O is not None:
            r0, r1 = oracle_mul_relin_moddown(O, ch, xs[i][0], xs[i][1], xs[i][0], xs[i][1], S_in, S, p, ea, eb)
            assert rows_equal(A0[i].download(S), r0, S) and rows_equal(A1[i].download(S), r1, S), i
    return ran, (A0, A1), (SA, EB)


@pytest.mark.parametrize("cfg, S_in_kind, ndrop, p, seeded", [
    ((8192, 257, 1, 119, 2), "ctxt", 1, 257, False),
    ((8192, 257, 1, 119, 2), "ctxt", 0, 257, True),
    ((8192, -1, 1, 240, 2), "ctxt", 2, 1, True),
    ((8192, 257, 1, 119, 2), "ctxt", 1, 2, False),
    ((8192, 257, 1, 119, 2), "ctxt+special", 1, 257, True),
], ids=["bgv-drop1", "bgv-nodrop-seeded", "ckks-drop2-seeded", "p2-drop1", "special-dropped-seeded"])
def test_square_relin_moddown_matches_oracle_and_multiply(closing, lib, cfg, S_in_kind, ndrop, p, seeded):
    ch, psis, O, E = make(lib, *cfg, nthreads=8)
    closing(E)
    S_in = sorted(ch.ctxt + ch.special) if S_in_kind == "ctxt+special" else ch.ctxt
    S = ch.ctxt[:len(ch.ctxt) - ndrop]
    ran, ops, key = square_case(E, ch, O, S_in, S, p, 3, seeded)
    if ndrop or S_in_kind != "ctxt":
        assert "k1_fwd_blk_square" in ran and "k1_tensor" not in ran, ran
    else:
        assert "k1_tensor" in ran and "k1_fwd_blk_square" not in ran, ran
    # a second call of the same shape allocates nothing
    before = E.stats()["device_bytes"]
    E.square_relin_moddown(*ops, S, S, p, *key)
    assert E.stats()["device_bytes"] == before


def test_square_relin_moddown_across_chunks(closing, lib, monkeypatch):
    """HB_CHUNK = 2: five items run as chunks of two, one and the scratch of the first chunk re-used."""
    monkeypatch.setenv("HB_CHUNK", "2")
    ch, psis, O, E = make(lib, 8192, 257, 1, 119, 2)
    closing(E)
    ran, *_ = square_case(E, ch, O, ch.ctxt, ch.ctxt[:-1], 257, 5, False, rng_seed=304)
    assert ran["k1_fwd_blk_square"] == 5, ran   # one item per chunk of the fused pass (two parts of a chunk of two slots)


@pytest.mark.parametrize("case", ["general-m", "force-v0"])
def test_square_relin_moddown_generic_paths(closing, sim_lib, monkeypatch, case):
    """General m (m = 105, p = 2) and HB_FORCE_V0: bit for bit hb_mul_relin_moddown on (x, copy of x)."""
    if case == "force-v0":
        monkeypatch.setenv("HB_FORCE_V0", "1")
        ch, psis, O, E = make(sim_lib, 8192, 257, 1, 119, 2)
        closing(E)
    else:
        ch = po.build_mod_chain(105, 2, 1, 120, 2)
        O, E = None, Engine(105, ch.primes, None, ch.digits, ch.special, lib=sim_lib)
        closing(E)
    ran, *_ = square_case(E, ch, O, ch.ctxt, ch.ctxt[:-1], ptxt_space(ch), 2, False, rng_seed=305)
    assert "k1_fwd_blk_square" not in ran and "k_pw_tensor" in ran, ran


@pytest.mark.gpu
@pytest.mark.parametrize("cfg, p", [((1 << 17, -1, 1, 1190, 2), 1), ((1 << 17, 257, 1, 1190, 2), 257)],
                         ids=["config2-ckks", "config3-bgv"])
def test_square_relin_moddown_full_size(closing, cuda_lib, cfg, p):
    """BASELINE configs 2 and 3's rings (m = 2^17, 20 ctxt primes): four squares, one prime dropped."""
    ch, psis, O, E = make(cuda_lib, *cfg, nthreads=8)
    closing(E)
    assert len(ch.ctxt) == 20
    ran, *_ = square_case(E, ch, O, ch.ctxt, ch.ctxt[:-1], p, 4, True, rng_seed=306)
    assert "k1_fwd_blk_square" in ran, ran


# ---- 3. worst-case words at the largest primes below 2^60

@pytest.mark.parametrize("case", [("sp", 257, 1), ("sp", -1, 2), ("gen", 2, 1), ("gen", -1, 1)],
                         ids=lambda c: "-".join(str(x) for x in c))
def test_square_relin_moddown_worst_case_words(closing, lib, case):
    """Operands at the top of their ranges (rows of q-1, alternating 0 / q-1, and coefficient extremes around q/2) on chains
    of the largest primes of both modulus forms, N = 2^16, keys of q-1.  Bounds: the subscale epilogue's
    (old - x + 12q) * P^-1 in [0, 4q) with x < 8q + 2^32 and old < 4q, then a0'^2, 2*a0'*a1' and a1'^2 below 2^125 in 128 bits."""
    form, p, ndrop = case
    ch, O, E = top_chain(lib, 1 << 17, p, form, [1, 1, 2], 2)
    closing(E)
    S_in = ch.ctxt
    S = S_in[:len(S_in) - ndrop]
    pt = 1 if p == -1 else p
    ea, EA = top_keys(ch, E)
    ops = [[operand(ch, O, S_in, k) for k in ks] for ks in (("top", "calt"), ("cmid", "top"), ("alt", "ctop"))]
    A0, A1 = ([E.poly(o[k], S_in) for o in ops] for k in range(2))
    E.profile(True)
    E.square_relin_moddown(A0, A1, S_in, S, pt, EA, EA)
    E.profile(False)
    ran = kernels(E)
    assert "k1_fwd_blk_square" in ran, ran
    for i, o in enumerate(ops):
        r0, r1 = oracle_mul_relin_moddown(O, ch, o[0], o[1], o[0], o[1], S_in, S, pt, ea, ea)
        assert rows_equal(A0[i].download(S), r0, S) and rows_equal(A1[i].download(S), r1, S), i


# ---- 4. argument errors: the code, and nothing launched

def test_errors_are_reported_before_any_launch(closing, lib):
    ch, psis, O, E = make(lib, 8192, 257, 1, 119, 2)
    closing(E)
    rng = np.random.default_rng(307)
    S = ch.ctxt
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    EA = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    EB = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    SA = E.seeded(nd, full, SEED)
    a0, a1, b0, b1 = (E.poly(rand(ch, rng, S, E.N), S) for _ in range(4))
    o2 = E.poly()

    def expect(code, f):
        E.profile(True)
        with pytest.raises(HbError) as e:
            f()
        E.profile(False)
        assert e.value.code == code, e.value
        assert E.profile_results() == [], E.profile_results()

    sq = lambda x0, x1, S_in=S, S_=S[:-1], ea=EA, eb=EB: E.square_relin_moddown(x0, x1, S_in, S_, 257, ea, eb)
    st = lambda x0, x1, y2, S_in=S, S_=S[:-1], norms=False: E.square_tensor(x0, x1, y2, S_in, S_, 257, norms)
    expect(HB_ERR_BAD_ARG, lambda: sq([], []))
    expect(HB_ERR_BAD_ARG, lambda: st([], [], []))
    expect(HB_ERR_BAD_ARG, lambda: sq([a0], [a0]))                       # one poly as both parts
    expect(HB_ERR_BAD_ARG, lambda: sq([a0, b0], [a1, a0]))               # one poly in two items
    expect(HB_ERR_BAD_ARG, lambda: st([a0], [a0], [o2], norms=True))
    expect(HB_ERR_BAD_ARG, lambda: st([a0], [a1], [a1]))                 # o2 aliasing an operand
    expect(HB_ERR_BAD_ARG, lambda: st([a0, b0], [a1, b1], [o2, o2]))     # o2 given twice
    expect(HB_ERR_BAD_ARG, lambda: sq([a0], [a1], S_=S, ea=EA[:1], eb=EB[:1]))   # too few key columns (S has two digits)
    expect(HB_ERR_BAD_ARG, lambda: sq([a0], [EB[0]]))                    # an operand aliasing a key
    expect(HB_ERR_BAD_ARG, lambda: sq([a0], [SA[0]]))                    # a seeded handle outside evk_a
    expect(HB_ERR_BAD_ARG, lambda: st([a0], [a1], [SA[0]]))
    expect(HB_ERR_INDEX_SET, lambda: sq([a0], [a1], S_in=S[:-1], S_=S))  # S not within S_in
    expect(HB_ERR_INDEX_SET, lambda: st([a0], [a1], [o2], S_in=S[:-1], S_=S))
    expect(HB_ERR_INDEX_SET, lambda: sq([a0], [a1], S_in=full, S_=[ch.special[0]]))   # S not within the ctxt primes
    # hb_mul_relin_moddown: an operand poly repeated among its 4*nitems operands
    mul = lambda x0, x1, y0, y1: E.mul_relin_moddown(x0, x1, y0, y1, S, S[:-1], 257, EA, EB)
    expect(HB_ERR_BAD_ARG, lambda: mul([a0], [a1], [a0], [a1]))
    expect(HB_ERR_BAD_ARG, lambda: mul([a0, b0], [a1, b1], [b0, o2], [b1, a1]))
    # no special primes
    ch2 = po.build_mod_chain(8192, 257, 1, 119, 2)
    E2 = closing(Engine(8192, ch2.primes, [po.find_psi(q, 8192) for q in ch2.primes], ch2.digits, [], lib=lib))
    x0, x1 = E2.poly(rand(ch2, rng, ch2.ctxt, E2.N), ch2.ctxt), E2.poly(rand(ch2, rng, ch2.ctxt, E2.N), ch2.ctxt)
    E2.profile(True)
    with pytest.raises(HbError) as e:
        E2.square_relin_moddown([x0], [x1], ch2.ctxt, ch2.ctxt[:-1], 257, [E2.poly()], [E2.poly()])
    E2.profile(False)
    assert e.value.code == HB_ERR_BAD_ARG and E2.profile_results() == []


# ---- 5. code generation on sm_90a

def test_square_kernel_has_no_local_array_stack_frame_or_spill(tmp_path):
    """k1_fwd_blk_square keeps its residues and second-pass twiddles in registers and a0' in shared memory: no local
    array in the PTX, and a (0, 0, 0) frame in `ptxas -v` for both instantiations."""
    nvcc = _nvcc()
    ptx = str(tmp_path / "hb_engine.ptx")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx",
                    os.path.join(CSRC, "hb_engine.cu"), "-o", ptx], check=True, capture_output=True, text=True)
    r = subprocess.run([os.path.join(os.path.dirname(nvcc), "ptxas"), "-arch=sm_90a", "-O3", "-v", ptx,
                        "-o", str(tmp_path / "hb_engine.cubin")], check=True, capture_output=True, text=True)
    mine = lambda k: re.match(r"_Z\d+k1_fwd_blk_squareI", k) is not None
    depots = {k: v for k, v in _depots(open(ptx).read()).items() if mine(k)}
    frames = {k: v for k, v in _frames(r.stdout + r.stderr).items() if mine(k)}
    assert len(frames) == 2, frames
    assert not depots, depots
    assert all(v == (0, 0, 0) for v in frames.values()), frames


# ---- 6. the C++ mirror (tests/cpp/test_square.cpp): square, power, cube, multiplyBy2 against the transcribed HElib code

def test_mirror_square_on_simulator():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_square", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "square OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_square_on_gpu():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_square")], capture_output=True, text=True)
    assert r.returncode == 0 and "square OK" in r.stdout, r.stdout + r.stderr
