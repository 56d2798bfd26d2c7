"""Hoisted linear maps (hb_hoisted_linear_map, SURVEY 8f-1): sum_j consts[j] * BasicAutomorphPrecon::automorph(k[j]) over
S | special in one pass -- the loop body of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252).

Checked bit for bit against the oracle doing the composed steps (automorph of every digit and of c0, addPrimesAndScale,
keySwitchDigits, pointwise multiply and add), against the composed engine path at full size, with seeded matrices, and
for its argument errors.  Unless marked, each test runs on the CPU simulator build and, marked gpu, on the H100.
"""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import make
from helib_b200.engine import Engine
from prg_sim import drop_stale_sim_build
from test_codegen import _depots, _frames, engine_codegen  # noqa: F401  (module-scoped compile fixture)
from test_cpp_shim import build_exe

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
HB_MAXB = 64
POW2 = [(64, 257, 1, 120, 2), (2048, 17, 2, 150, 3), (4096, 257, 1, 60, 2), (8192, -1, 1, 119, 2)]
GEN = [(45, 2, 1, 100, 2), (105, 2, 1, 120, 2), (1285, 2, 1, 120, 2)]


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


class GenOracle:
    """The composed steps for general m, restated on dense [nprimes][phi(m)] arrays: sigma_k(x)[j] = x[idx(rep(j)*k mod m)]
    (src/DoubleCRT.cpp:1160-1202) and row-wise modular arithmetic in Python integers."""

    def __init__(self, ch):
        self.m, self.N, self.primes, self.special = ch.m, ch.phim, ch.primes, ch.special
        self.rep = po.zms_rep(ch.m)
        self.pos = {r: i for i, r in enumerate(self.rep)}

    def zeros(self):
        return np.zeros((len(self.primes), self.N), dtype=np.uint64)

    def _row(self, data, i, vals):
        data[i] = np.array([int(v) for v in vals], dtype=np.uint64)

    def automorph(self, data, idx, k):
        perm = np.array([self.pos[r * k % self.m] for r in self.rep])
        for i in idx:
            data[i] = data[i][perm]

    def add_primes_and_scale(self, data, S, add):
        P = math.prod(self.primes[i] for i in add)
        for i in S:
            q = self.primes[i]
            self._row(data, i, data[i].astype(object) * (P % q) % q)
        for i in add:
            data[i] = 0

    def keyswitch_digits(self, digits, idx, evk_a, evk_b, out0, out1):
        for i in idx:
            q = self.primes[i]
            s0, s1 = out0[i].astype(object), out1[i].astype(object)
            for d in range(digits.shape[0]):
                s0 = s0 + digits[d][i].astype(object) * evk_b[d][i].astype(object)
                s1 = s1 + digits[d][i].astype(object) * evk_a[d][i].astype(object)
            self._row(out0, i, s0 % q)
            self._row(out1, i, s1 % q)

    def pointwise(self, op, dst, src, idx):
        for i in idx:
            q = self.primes[i]
            a, b = dst[i].astype(object), src[i].astype(object)
            self._row(dst, i, (a * b if op == "mul" else a + b) % q)


def _setup(lib, cfg):
    m = cfg[0]
    if m & (m - 1) == 0:
        ch, psis, O, E = make(lib, *cfg)
        return ch, O, E
    ch = po.build_mod_chain(*cfg)
    return ch, GenOracle(ch), Engine(m, ch.primes, None, ch.digits, ch.special, lib=lib)


def _rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def _reference(O, ch, dig, c0, c1, ks, cs, ea, eb, acc0, acc1):
    """acc += sum_j cs[j] * automorph_j, step by step (BasicAutomorphPrecon::automorph, multByConstant, addCtxt)."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    acc0, acc1 = acc0.copy(), acc1.copy()
    for j, k in enumerate(ks):
        r0 = c0.copy()
        if k == 1:
            r1 = c1.copy()
            O.add_primes_and_scale(r0, S, ch.special)
            O.add_primes_and_scale(r1, S, ch.special)
        else:
            O.automorph(r0, S, k)
            O.add_primes_and_scale(r0, S, ch.special)
            r1 = O.zeros()
            rd = dig.copy()
            for i in range(rd.shape[0]):
                O.automorph(rd[i], Sp, k)
            O.keyswitch_digits(rd, Sp, ea[j], eb[j], r0, r1)
        O.pointwise("mul", r0, cs[j], Sp)
        O.pointwise("mul", r1, cs[j], Sp)
        O.pointwise("add", acc0, r0, Sp)
        O.pointwise("add", acc1, r1, Sp)
    return acc0, acc1


def _units(m, n):
    return [t for t in range(2, m - 1) if math.gcd(t, m) == 1][:n]


def _check(lib, cfg, ks, nitems=2, accumulate=False, seed=0):
    ch, O, E = _setup(lib, cfg)
    rng = np.random.default_rng(seed)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    namt = len(ks)
    dig = [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) for _ in range(nitems)]
    c0 = [_rand(ch, rng, S, N) for _ in range(nitems)]
    c1 = [_rand(ch, rng, S, N) for _ in range(nitems)]
    ea = [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) for _ in range(namt)]
    eb = [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) for _ in range(namt)]
    cs = [_rand(ch, rng, Sp, N) for _ in range(namt)]
    a0 = [_rand(ch, rng, Sp, N) if accumulate else O.zeros() for _ in range(nitems)]
    a1 = [_rand(ch, rng, Sp, N) if accumulate else O.zeros() for _ in range(nitems)]
    D = [[E.poly(d[i], Sp) for i in range(nd)] for d in dig]
    C0 = [E.poly(x, S) for x in c0]
    C1 = [E.poly(x, S) for x in c1]
    EA = [[E.poly(x[i], Sp) for i in range(nd)] if k != 1 else None for x, k in zip(ea, ks)]
    EB = [[E.poly(x[i], Sp) for i in range(nd)] if k != 1 else None for x, k in zip(eb, ks)]
    CS = [E.poly(x, Sp) for x in cs]
    A0 = [E.poly(x, Sp) if accumulate else E.poly(_rand(ch, rng, Sp, N), Sp) for x in a0]   # overwritten when not accumulating
    A1 = [E.poly(x, Sp) if accumulate else E.poly(_rand(ch, rng, Sp, N), Sp) for x in a1]
    E.hoisted_linear_map(D, S, C0, C1, ks, CS, EA, EB, A0, A1, accumulate=accumulate)
    for it in range(nitems):
        r0, r1 = _reference(O, ch, dig[it], c0[it], c1[it], ks, cs, ea, eb, a0[it], a1[it])
        assert (A0[it].download(Sp)[Sp] == r0[Sp]).all() and (A1[it].download(Sp)[Sp] == r1[Sp]).all(), (cfg, it)
    E.close()


# ---- 1. parity with the oracle

@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("cfg", POW2 + GEN)
def test_matches_the_composed_steps(lib, cfg, accumulate):
    """k = 1, k = m - 1, a repeated amount and two others, over power-of-two and general rings."""
    m = cfg[0]
    u = _units(m, 2)
    _check(lib, cfg, [1, m - 1, u[0], u[0], u[1]], nitems=2, accumulate=accumulate, seed=m + accumulate)


def test_amounts_across_the_launch_cap(lib):
    """70 amounts: two launches per item chunk, the second accumulating on the first."""
    m = 64
    u = _units(m, 30)
    ks = [u[j % len(u)] for j in range(69)] + [1]
    _check(lib, (64, 257, 1, 120, 2), ks, nitems=3, accumulate=True, seed=70)


def test_items_across_the_batch_cap(lib):
    _check(lib, (64, 257, 1, 120, 2), [1, 3, 63], nitems=HB_MAXB + 3, seed=67)


def test_general_m_items_across_the_batch_cap(lib):
    _check(lib, (45, 2, 1, 100, 2), [44, 2], nitems=HB_MAXB + 1, accumulate=True, seed=45)


# ---- 2. seeded matrices

def _seeded_case(E, ch, rng, namt, nitems=2):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    ks = [_units(ch.m, namt)[j % len(_units(ch.m, namt))] for j in range(namt)]
    D = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(nitems)]
    C0 = [E.poly(_rand(ch, rng, S, N), S) for _ in range(nitems)]
    CS = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(namt)]
    EB = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(namt)]
    return ks, D, C0, CS, EB


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (105, 2, 1, 120, 2)])
def test_seeded_expanded_and_mixed_matrices_agree(lib, cfg):
    ch, O, E = _setup(lib, cfg)
    rng = np.random.default_rng(5)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, namt = len(ch.digits), 12
    ks, D, C0, CS, EB = _seeded_case(E, ch, rng, namt)
    seeded = [E.seeded(nd, Sp, 1000 + j) for j in range(namt)]
    expanded = []
    for j in range(namt):
        P = [E.poly() for _ in range(nd)]
        E.randomize(P, Sp, 1000 + j)
        expanded.append(P)
    mixed = [seeded[j] if j % 2 else expanded[j] for j in range(namt)]
    outs = []
    for EA in (expanded, seeded, mixed):
        A0, A1 = [E.poly() for _ in D], [E.poly() for _ in D]
        E.hoisted_linear_map(D, S, C0, None, ks, CS, EA, EB, A0, A1)
        outs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[1]))
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[2]))
    E.close()


def test_seeded_scratch_does_not_grow_with_the_amounts(sim_lib):
    ch, O, E = _setup(sim_lib, (64, 257, 1, 120, 2))
    rng = np.random.default_rng(6)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    ks, D, C0, CS, EB = _seeded_case(E, ch, rng, 64)
    EA = [E.seeded(nd, Sp, 77 + j) for j in range(64)]
    A0, A1 = [E.poly() for _ in D], [E.poly() for _ in D]
    E.hoisted_linear_map(D, S, C0, None, ks[:8], CS[:8], EA[:8], EB[:8], A0, A1)
    eight = E.stats()["device_bytes"]
    E.hoisted_linear_map(D, S, C0, None, ks, CS, EA, EB, A0, A1)
    assert E.stats()["device_bytes"] <= eight
    E.close()


# ---- 3. argument errors: each reported before any launch

_KEEP = []


def _pa(lst):
    a = (C.c_void_p * max(1, len(lst)))(*[None if p is None else p.h for p in lst])
    _KEEP.append(a)
    return a


def test_argument_errors_launch_nothing(sim_lib):
    ch, O, E = _setup(sim_lib, (64, 257, 1, 120, 2))
    rng = np.random.default_rng(8)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    L = E.lib
    D = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    c0, c1, cs = E.poly(_rand(ch, rng, S, N), S), E.poly(_rand(ch, rng, S, N), S), E.poly(_rand(ch, rng, Sp, N), Sp)
    EA = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    EB = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    a0, a1 = E.poly(), E.poly()
    X = E.seeded(1, Sp, 5)[0]
    short = E.seeded(nd, sorted(ch.ctxt[:-1] + ch.special), 6)    # lacks the top ctxt prime
    Sarr = np.ascontiguousarray(np.array(S, dtype=np.int32))
    Sbad = np.ascontiguousarray(np.array(S + ch.special[:1], dtype=np.int32))

    def call(digits=D, S_=Sarr, c0_=c0, c1_=c1, ks=(3,), consts=None, ea=EA, eb=EB, acc0=a0, acc1=a1, ndig=nd, maxdig=nd, namt=None):
        kk = np.ascontiguousarray(np.array(ks, dtype=np.uint64))
        consts = consts or [cs] * len(ks)
        namt = len(ks) if namt is None else namt
        return L.hb_hoisted_linear_map(_pa(digits), maxdig, ndig, 1, S_.ctypes.data_as(C.POINTER(C.c_int32)), len(S_), _pa([c0_]),
                                       _pa([c1_]) if c1_ is not None else None, namt, kk.ctypes.data_as(C.POINTER(C.c_uint64)),
                                       _pa(consts), _pa(list(ea) * len(ks)), _pa(list(eb) * len(ks)), _pa([acc0]), _pa([acc1]), 0)

    cases = [
        ("k = 2", HB_ERR_INDEX_SET, lambda: call(ks=(3, 2))),
        ("k = 0", HB_ERR_INDEX_SET, lambda: call(ks=(0,))),
        ("k = m", HB_ERR_INDEX_SET, lambda: call(ks=(64,))),
        ("S with a special prime", HB_ERR_INDEX_SET, lambda: call(S_=Sbad)),
        ("seeded evk_a without a needed row", HB_ERR_INDEX_SET, lambda: call(ea=short)),
        ("namt = 0", HB_ERR_BAD_ARG, lambda: call(namt=0)),
        ("ndig = 0", HB_ERR_BAD_ARG, lambda: call(ndig=0)),
        ("ndig > maxdig", HB_ERR_BAD_ARG, lambda: call(ndig=nd + 1)),
        ("c1 NULL with k = 1", HB_ERR_BAD_ARG, lambda: call(ks=(3, 1), c1_=None)),
        ("acc0 = a digit", HB_ERR_BAD_ARG, lambda: call(acc0=D[0])),
        ("acc1 = c0", HB_ERR_BAD_ARG, lambda: call(acc1=c0)),
        ("acc0 = c1", HB_ERR_BAD_ARG, lambda: call(acc0=c1)),
        ("acc1 = a constant", HB_ERR_BAD_ARG, lambda: call(acc1=cs)),
        ("acc0 = acc1", HB_ERR_BAD_ARG, lambda: call(acc1=a0)),
        ("seeded digit", HB_ERR_BAD_ARG, lambda: call(digits=[X] + D[1:])),
        ("seeded c0", HB_ERR_BAD_ARG, lambda: call(c0_=X)),
        ("seeded c1", HB_ERR_BAD_ARG, lambda: call(c1_=X)),
        ("seeded constant", HB_ERR_BAD_ARG, lambda: call(consts=[X])),
        ("seeded evk_b", HB_ERR_BAD_ARG, lambda: call(eb=[X] + EB[1:])),
        ("seeded acc0", HB_ERR_BAD_ARG, lambda: call(acc0=X)),
        ("seeded acc1", HB_ERR_BAD_ARG, lambda: call(acc1=X)),
    ]
    assert call() == 0
    for name, code, f in cases:
        E.sync()
        before = E.stats()["launches"]
        rc = f()
        assert rc == code, (name, rc, L.hb_last_error())
        assert E.stats()["launches"] == before, name
    # k = 1 ignores its matrix, which may be NULL
    kk = np.array([1], dtype=np.uint64)
    rc = L.hb_hoisted_linear_map(_pa(D), nd, nd, 1, Sarr.ctypes.data_as(C.POINTER(C.c_int32)), len(Sarr), _pa([c0]), _pa([c1]), 1,
                                 kk.ctypes.data_as(C.POINTER(C.c_uint64)), _pa([cs]), None, None, _pa([a0]), _pa([a1]), 0)
    assert rc == 0, L.hb_last_error()
    E.close()


# ---- 4. code generation

def test_linear_map_kernel_keeps_its_state_in_registers(engine_codegen):
    ptx, report = engine_codegen
    frames = {k: v for k, v in _frames(report).items() if "k_ks_linmap" in k}
    assert len(frames) == 3, frames
    assert all(v == (0, 0, 0) for v in frames.values()), frames
    assert not {k: v for k, v in _depots(ptx).items() if "k_ks_linmap" in k}


# ---- 5. the C++ mirror (tests/cpp/test_linear_map.cpp): BasicAutomorphPrecon::linearCombination

def test_mirror_linear_combination_on_simulator():
    r = subprocess.run([build_exe("test_linear_map", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "linear map OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_linear_combination_on_gpu():
    r = subprocess.run([build_exe("test_linear_map")], capture_output=True, text=True)
    assert r.returncode == 0 and "linear map OK" in r.stdout, r.stdout + r.stderr


# ---- 6. full size on the GPU: parity with the composed engine path, seeded keys, CUDA graph

def _full(cuda_lib, m, p, bits, c):
    from helib_b200 import Chain
    ch = Chain(m, p, 1, bits, c, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    return ch, E


def _composed(E, digs, S, C0, ks, CS, EA, EB, A0, A1, T0, T1):
    """hb_automorph_keyswitch_digits + hb_pointwise MUL + ADD per amount."""
    Sp = sorted(S + E.special)
    for j, k in enumerate(ks):
        o0, o1 = (A0, A1) if j == 0 else (T0, T1)
        E.automorph_keyswitch_digits(digs, S, C0, k, EA[j], EB[j], o0, o1)
        E.pointwise("mul", o0 + o1, [CS[j]] * (2 * len(o0)), Sp)
        if j:
            E.pointwise("add", A0 + A1, T0 + T1, Sp)


@pytest.mark.gpu
@pytest.mark.parametrize("ring", ["cfg3", "cfg5"])
def test_full_size_matches_the_composed_engine_path(cuda_lib, ring):
    """Config 3's ring (BGV m = 2^17, 26 ctxt + 9 special primes, 3 digits) and config 5's (m = 21845, Bluestein rows):
    the fused call equals hb_automorph_keyswitch_digits + MUL + ADD bit for bit, with expanded and with seeded matrices."""
    ch, E = _full(cuda_lib, *((1 << 17, 257, 1500, 3) if ring == "cfg3" else (21845, 2, 580, 2)))
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, B = len(ch.digits), 3
    ks = _units(ch.m, 3) + [_units(ch.m, 1)[0], ch.m - 1]
    C0, C1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.randomize(C0 + C1, S, 11)
    digs = E.break_into_digits(C1, S)
    CS = [E.poly() for _ in ks]
    E.randomize(CS, Sp, 12)
    EB = [[E.poly() for _ in range(nd)] for _ in ks]
    E.randomize([x for m_ in EB for x in m_], Sp, 13)
    EA = [[E.poly() for _ in range(nd)] for _ in ks]
    for j, m_ in enumerate(EA):
        E.randomize(m_, Sp, 100 + j)
    SA = [E.seeded(nd, Sp, 100 + j) for j in range(len(ks))]
    R0, R1, T0, T1 = ([E.poly() for _ in range(B)] for _ in range(4))
    _composed(E, digs, S, C0, ks, CS, EA, EB, R0, R1, T0, T1)
    ref = [x.download(Sp)[Sp] for x in R0 + R1]
    for keys in (EA, SA):
        A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        E.hoisted_linear_map(digs, S, C0, C1, ks, CS, keys, EB, A0, A1)
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(ref, A0 + A1))
    E.close()


@pytest.mark.gpu
def test_config3_seeded_call_in_a_cuda_graph(cuda_lib):
    import torch
    ch, E = _full(cuda_lib, 1 << 17, 257, 1500, 3)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, B = len(ch.digits), 2
    ks = _units(ch.m, 6)
    C0, C1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.randomize(C0 + C1, S, 21)
    digs = E.break_into_digits(C1, S)
    CS = [E.poly() for _ in ks]
    E.randomize(CS, Sp, 22)
    EB = [[E.poly() for _ in range(nd)] for _ in ks]
    E.randomize([x for m_ in EB for x in m_], Sp, 23)
    SA = [E.seeded(nd, Sp, 200 + j) for j in range(len(ks))]
    A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.hoisted_linear_map(digs, S, C0, C1, ks, CS, SA, EB, A0, A1)
    ref = [x.download(Sp)[Sp] for x in A0 + A1]
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    E.set_stream(side.cuda_stream)
    E.hoisted_linear_map(digs, S, C0, C1, ks, CS, SA, EB, A0, A1)   # warm on the capturing stream
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        E.hoisted_linear_map(digs, S, C0, C1, ks, CS, SA, EB, A0, A1)
    for _ in range(2):
        for x in A0 + A1:
            x.upload(np.zeros((E.np, E.N), dtype=np.uint64), Sp)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(ref, A0 + A1))
    torch.cuda.set_stream(torch.cuda.default_stream())
    E.close()
