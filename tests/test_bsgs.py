"""BSGS linear maps (hb_bsgs_linear_map, SURVEY 8f-1): the giant-step phase of MatMul1DExec::mul's non-iterative
baby-step/giant-step branches (src/matmul.cpp:1022-1057 native, 1097-1142 bad dimension).

Checked bit for bit against the oracle doing HElib's steps one by one (MulAdd over the baby steps, then per giant step
automorph, the mod-down of reLinearize in the extended form, breakIntoDigits, addPrimesAndScale and keySwitchDigits, and
the adds), against the composed engine path at full size, with seeded matrices, and for its argument errors.  Unless
marked, each test runs on the CPU simulator build and, marked gpu, on the H100.
"""
import ctypes as C
import subprocess

import numpy as np
import pytest

import pyoracle as po
from bench_bsgs import composed, gen_of
from common import make
from helib_b200.engine import Engine
from prg_sim import drop_stale_sim_build
from test_codegen import _depots, _frames, engine_codegen  # noqa: F401  (module-scoped compile fixture)
from test_cpp_shim import build_exe

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
HB_MAXB = 64
POW2 = [(64, 257, 1, 120, 2), (2048, 17, 2, 150, 3), (8192, -1, 1, 119, 2)]
GEN = [(45, 2, 1, 100, 2), (105, 2, 1, 120, 2), (1285, 2, 1, 120, 2)]


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


class PowOps:
    """HElib's DoubleCRT steps on dense [nprimes][N] arrays, power-of-two m: the C++ oracle."""

    def __init__(self, O, ch):
        self.O, self.ch = O, ch

    def zeros(self):
        return self.O.zeros()

    def muladd(self, dst, a, b, idx):
        t = a.copy()
        self.O.pointwise("mul", t, b, idx)
        self.O.pointwise("add", dst, t, idx)

    def scale(self, x, idx, f):
        self.O.scale_by_word(x, idx, f)

    def add(self, dst, src, idx):
        self.O.pointwise("add", dst, src, idx)

    def automorph(self, x, idx, k):
        self.O.automorph(x, idx, k)

    def add_primes_and_scale(self, x, S, add):
        self.O.add_primes_and_scale(x, S, add)

    def scale_down(self, x, cur, keep, p):
        self.O.scale_down(x, cur, keep, p)

    def break_into_digits(self, x, S):
        return list(self.O.break_into_digits(x, S))

    def keyswitch_digits(self, digs, idx, ea, eb, out0, out1):
        self.O.keyswitch_digits(np.stack(digs), idx, ea, eb, out0, out1)


class GenOps(PowOps):
    """The same steps for general m, on the big-integer Python oracle (pyoracle.PyDCRT, Bluestein rows)."""

    def __init__(self, ch, roots):
        self.ch, self.roots = ch, roots

    def zeros(self):
        return np.zeros((len(self.ch.primes), self.ch.phim), dtype=np.uint64)

    def _d(self, x, idx):
        return po.PyDCRT(self.ch, self.roots, {i: [int(v) for v in x[i]] for i in idx})

    def _put(self, x, d):
        for i, r in d.rows.items():
            x[i] = np.array(r, dtype=np.uint64)

    def _rows(self, f, dst, src, idx):
        for i in idx:
            q = self.ch.primes[i]
            dst[i] = np.array([f(int(a), int(b)) % q for a, b in zip(dst[i], src[i])], dtype=np.uint64)

    def muladd(self, dst, a, b, idx):
        t = a.copy()
        self._rows(lambda u, v: u * v, t, b, idx)
        self._rows(lambda u, v: u + v, dst, t, idx)

    def scale(self, x, idx, f):
        for i in idx:
            q = self.ch.primes[i]
            x[i] = np.array([int(v) * f % q for v in x[i]], dtype=np.uint64)

    def add(self, dst, src, idx):
        self._rows(lambda u, v: u + v, dst, src, idx)

    def automorph(self, x, idx, k):
        self._put(x, self._d(x, idx).automorph(k))

    def add_primes_and_scale(self, x, S, add):
        self._put(x, self._d(x, S).add_primes_and_scale(add))

    def scale_down(self, x, cur, keep, p):
        d = self._d(x, cur)
        d.scale_down_to_set(keep, p)
        self._put(x, d)

    def break_into_digits(self, x, S):
        out = []
        for d in self._d(x, S).break_into_digits()[0]:
            y = self.zeros()
            self._put(y, d)
            out.append(y)
        return out

    def keyswitch_digits(self, digs, idx, ea, eb, out0, out1):
        for d, a, b in zip(digs, ea, eb):
            t0, t1 = d.copy(), d.copy()
            self._rows(lambda u, v: u * v, t0, b, idx)
            self._rows(lambda u, v: u * v, t1, a, idx)
            self.add(out0, t0, idx)
            self.add(out1, t1, idx)


def _setup(lib, cfg):
    m = cfg[0]
    if m & (m - 1) == 0:
        ch, psis, O, E = make(lib, *cfg)
        return ch, PowOps(O, ch), E
    ch = po.build_mod_chain(*cfg)
    E = Engine(m, ch.primes, None, ch.digits, ch.special, lib=lib)
    return ch, GenOps(ch, [po.cmod_root(q, m) for q in ch.primes]), E


def _ptxt(ch):
    return 1 if ch.p == -1 else ch.p ** ch.r


def _rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def _reference(X, ch, b0, b1, cs, ks, scal, extended, ea, eb, acc0, acc1):
    """The giant steps of MatMul1DExec::mul's BSGS loop, step by step: acc_inner = MulAdd over the baby steps; for k > 0
    acc_inner.smartAutomorph (automorph, [dropSmallAndSpecialPrimes], relin_CKKS_adjust, keySwitchPart); acc += acc_inner."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    R = Sp if extended else S
    p = _ptxt(ch)
    acc0, acc1 = acc0.copy(), acc1.copy()
    for t, k in enumerate(ks):
        x0, x1 = X.zeros(), X.zeros()
        for j, c in enumerate(cs[t]):
            if c is not None:
                X.muladd(x0, b0[j], c, R)
                X.muladd(x1, b1[j], c, R)
        f = scal[t] if scal is not None else 1
        if k == 1:
            if f != 1:    # the ABI's scal[t] multiplies every giant step's sum; a caller passes 1 where HElib has no reLinearize
                X.scale(x0, R, f)
                X.scale(x1, R, f)
            if not extended:
                X.add_primes_and_scale(x0, S, ch.special)
                X.add_primes_and_scale(x1, S, ch.special)
            X.add(acc0, x0, Sp)
            X.add(acc1, x1, Sp)
            continue
        X.automorph(x0, R, k)
        X.automorph(x1, R, k)
        if extended:
            X.scale_down(x0, Sp, S, p)
            X.scale_down(x1, Sp, S, p)
        if f != 1:
            X.scale(x0, S, f)
            X.scale(x1, S, f)
        digs = X.break_into_digits(x1, S)
        r0, r1 = x0.copy(), X.zeros()
        X.add_primes_and_scale(r0, S, ch.special)
        X.keyswitch_digits(digs, Sp, ea[t], eb[t], r0, r1)
        X.add(acc0, r0, Sp)
        X.add(acc1, r1, Sp)
    return acc0, acc1


def _giant(m, g, h):
    gen = gen_of(m)
    return [pow(gen, g * t, m) for t in range(h)]


def _check(lib, cfg, nbaby, ks, extended=False, nitems=2, scal=None, zero=(), accumulate=False, seed=0, cs_per=None):
    """cs_per[t]: the number of nonzero diagonals of giant step t (the rest None); zero: (t, j) pairs left None."""
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(seed)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    R = Sp if extended else S
    nd, N, ng = len(ch.digits), E.N, len(ks)
    b0 = [[_rand(ch, rng, R, N) for _ in range(nbaby)] for _ in range(nitems)]
    b1 = [[_rand(ch, rng, R, N) for _ in range(nbaby)] for _ in range(nitems)]
    cs = [[None if (t, j) in zero or (cs_per and j >= cs_per[t]) else _rand(ch, rng, R, N) for j in range(nbaby)] for t in range(ng)]
    ea = [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) for _ in range(ng)]
    eb = [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) for _ in range(ng)]
    a0 = [_rand(ch, rng, Sp, N) if accumulate else X.zeros() for _ in range(nitems)]
    a1 = [_rand(ch, rng, Sp, N) if accumulate else X.zeros() for _ in range(nitems)]
    B0 = [[E.poly(x, R) for x in it] for it in b0]
    B1 = [[E.poly(x, R) for x in it] for it in b1]
    CS = [[E.poly(x, R) if x is not None else None for x in row] for row in cs]
    EA = [[E.poly(x[i], Sp) for i in range(nd)] if k != 1 else None for x, k in zip(ea, ks)]
    EB = [[E.poly(x[i], Sp) for i in range(nd)] if k != 1 else None for x, k in zip(eb, ks)]
    A0 = [E.poly(x, Sp) if accumulate else E.poly(_rand(ch, rng, Sp, N), Sp) for x in a0]   # overwritten when not accumulating
    A1 = [E.poly(x, Sp) if accumulate else E.poly(_rand(ch, rng, Sp, N), Sp) for x in a1]
    E.bsgs_linear_map(B0, B1, S, ks, CS, EA, EB, A0, A1, extended=extended, ptxt_space=_ptxt(ch), scal=scal, accumulate=accumulate)
    for it in range(nitems):
        r0, r1 = _reference(X, ch, b0[it], b1[it], cs, ks, scal, extended, ea, eb, a0[it], a1[it])
        assert (A0[it].download(Sp)[Sp] == r0[Sp]).all() and (A1[it].download(Sp)[Sp] == r1[Sp]).all(), (cfg, it)
    E.close()


# ---- 1. parity with the oracle

@pytest.mark.parametrize("extended", [0, 1], ids=["native", "extended"])
@pytest.mark.parametrize("cfg", POW2 + GEN)
def test_matches_the_composed_steps(lib, cfg, extended):
    """D = g^2 (g = h = 3; 2g baby steps in the extended form) with one zero diagonal; general m rings have p = 2, so the
    extended form's mod-down meets the tie rule."""
    m, g = cfg[0], 3
    nb = 2 * g if extended else g
    _check(lib, cfg, nb, _giant(m, g, 3), extended=extended, zero={(1, 1)}, seed=m + extended)


@pytest.mark.parametrize("cfg", [(64, 257, 1, 120, 2), (8192, -1, 1, 119, 2), (105, 2, 1, 120, 2)])
def test_scal_and_accumulate(lib, cfg):
    """relin_CKKS_adjust's factor on every giant step (native form), added to accumulators that hold data."""
    m = cfg[0]
    _check(lib, cfg, 3, _giant(m, 3, 3), scal=[7, 3, (1 << 40) + 5], accumulate=True, seed=7)


@pytest.mark.parametrize("extended", [0, 1], ids=["native", "extended"])
@pytest.mark.parametrize("cfg", [(64, 257, 1, 120, 2), (45, 2, 1, 100, 2)])
def test_short_last_giant_step(lib, cfg, extended):
    """D = 10, g = 4: h = 3 and the last giant step has two diagonals."""
    m, g = cfg[0], 4
    per = [4, 4, 2]
    nb = 2 * g if extended else g
    if extended:
        per = [2 * x for x in per]
    _check(lib, cfg, nb, _giant(m, g, 3), extended=extended, cs_per=per, seed=10 + extended)


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (105, 2, 1, 120, 2)])
def test_one_baby_step_and_one_giant_step(lib, cfg):
    m = cfg[0]
    _check(lib, cfg, 1, _giant(m, 1, 4), seed=1)                     # g = 1
    _check(lib, cfg, 5, [1], extended=1, seed=2)                      # h = 1: no rotation, no key switch


def test_giant_steps_across_groups(lib):
    """35 giant steps of one item and 12 of three: more than one group of 32 (giant step, item) pairs."""
    cfg = (64, 257, 1, 120, 2)
    _check(lib, cfg, 2, _giant(64, 2, 35), nitems=1, seed=35)
    _check(lib, cfg, 2, _giant(64, 2, 12), nitems=3, extended=1, accumulate=True, seed=12)


@pytest.mark.parametrize("nitems", [1, 2, 4])
def test_baby_steps_across_launches(lib, nitems):
    """250 baby steps: more than one k_bsgs_mac launch per pair, the later ones adding to the scattered sums."""
    _check(lib, (64, 257, 1, 120, 2), 250, _giant(64, 250, 2), nitems=nitems, seed=250 + nitems)


def test_items_across_the_batch_cap(lib):
    _check(lib, (64, 257, 1, 120, 2), 2, _giant(64, 2, 2), nitems=HB_MAXB + 2, seed=66)


def test_general_m_items_across_the_batch_cap(lib):
    _check(lib, (45, 2, 1, 100, 2), 2, _giant(45, 2, 2), nitems=HB_MAXB + 1, extended=1, seed=45)


def test_all_zero_diagonals_give_zero(lib):
    ch, X, E = _setup(lib, (64, 257, 1, 120, 2))
    rng = np.random.default_rng(3)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    B = [[E.poly(_rand(ch, rng, S, N), S) for _ in range(2)]]
    EA = [None, [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]]
    EB = [None, [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]]
    A0, A1 = [E.poly(_rand(ch, rng, Sp, N), Sp)], [E.poly(_rand(ch, rng, Sp, N), Sp)]
    E.bsgs_linear_map(B, B, S, [1, 5], [[None, None], [None, None]], EA, EB, A0, A1, ptxt_space=257)
    assert not A0[0].download(Sp)[Sp].any() and not A1[0].download(Sp)[Sp].any()
    E.close()


# ---- 2. seeded matrices

def _seeded_case(E, ch, rng, ng, nitems=2, nb=2):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    ks = _giant(ch.m, nb, ng)
    B0 = [[E.poly(_rand(ch, rng, S, N), S) for _ in range(nb)] for _ in range(nitems)]
    B1 = [[E.poly(_rand(ch, rng, S, N), S) for _ in range(nb)] for _ in range(nitems)]
    CS = [[E.poly(_rand(ch, rng, S, N), S) for _ in range(nb)] for _ in range(ng)]
    EB = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(ng)]
    return ks, B0, B1, CS, EB


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (105, 2, 1, 120, 2)])
def test_seeded_expanded_and_mixed_matrices_agree(lib, cfg):
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(5)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, ng = len(ch.digits), 10
    ks, B0, B1, CS, EB = _seeded_case(E, ch, rng, ng)
    seeded = [E.seeded(nd, Sp, 1000 + j) for j in range(ng)]
    expanded = []
    for j in range(ng):
        P = [E.poly() for _ in range(nd)]
        E.randomize(P, Sp, 1000 + j)
        expanded.append(P)
    mixed = [seeded[j] if j % 2 else expanded[j] for j in range(ng)]
    outs = []
    for EA in (expanded, seeded, mixed):
        A0, A1 = [E.poly() for _ in B0], [E.poly() for _ in B0]
        E.bsgs_linear_map(B0, B1, S, ks, CS, EA, EB, A0, A1, ptxt_space=_ptxt(ch))
        outs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[1]))
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[2]))
    E.close()


def test_scratch_does_not_grow_with_the_giant_steps(sim_lib):
    ch, X, E = _setup(sim_lib, (64, 257, 1, 120, 2))
    rng = np.random.default_rng(6)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    ks, B0, B1, CS, EB = _seeded_case(E, ch, rng, 40, nitems=1)
    EA = [E.seeded(nd, Sp, 77 + j) for j in range(40)]
    A0, A1 = [E.poly()], [E.poly()]
    E.bsgs_linear_map(B0, B1, S, ks[:32], CS[:32], EA[:32], EB[:32], A0, A1, ptxt_space=257)   # one full group
    full = E.stats()["device_bytes"]
    E.bsgs_linear_map(B0, B1, S, ks, CS, EA, EB, A0, A1, ptxt_space=257)
    assert E.stats()["device_bytes"] <= full
    E.close()


# ---- 3. argument errors: each reported before any launch

_KEEP = []


def _pa(lst):
    a = (C.c_void_p * max(1, len(lst)))(*[None if p is None else p.h for p in lst])
    _KEEP.append(a)
    return a


def test_argument_errors_launch_nothing(sim_lib):
    ch, X, E = _setup(sim_lib, (64, 257, 1, 120, 2))
    rng = np.random.default_rng(8)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    L = E.lib
    b0, b1 = [E.poly(_rand(ch, rng, S, N), S) for _ in range(2)], [E.poly(_rand(ch, rng, S, N), S) for _ in range(2)]
    cs = [E.poly(_rand(ch, rng, S, N), S) for _ in range(2)]
    EA = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    EB = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    a0, a1 = E.poly(), E.poly()
    Xs = E.seeded(1, Sp, 5)[0]
    short = E.seeded(nd, sorted(ch.ctxt[:-1] + ch.special), 6)    # lacks the top ctxt prime
    Sarr = np.ascontiguousarray(np.array(S, dtype=np.int32))
    Sbad = np.ascontiguousarray(np.array(S + ch.special[:1], dtype=np.int32))

    def call(B0=b0, B1=b1, nbaby=2, nitems=1, S_=Sarr, ext=0, p=257, ks=(1, 3), consts=None, scal=None, ea=EA, eb=EB,
             ndig=nd, acc0=a0, acc1=a1, ngiant=None):
        kk = np.ascontiguousarray(np.array(ks, dtype=np.uint64))
        consts = consts if consts is not None else cs * len(ks)
        ngiant = len(ks) if ngiant is None else ngiant
        sc = np.ascontiguousarray(np.array(scal, dtype=np.uint64)) if scal is not None else None
        return L.hb_bsgs_linear_map(_pa(B0), _pa(B1), nbaby, nitems, S_.ctypes.data_as(C.POINTER(C.c_int32)), len(S_), ext,
                                    C.c_uint64(p), ngiant, kk.ctypes.data_as(C.POINTER(C.c_uint64)), _pa(consts),
                                    sc.ctypes.data_as(C.POINTER(C.c_uint64)) if sc is not None else None,
                                    _pa(list(ea) * len(ks)), _pa(list(eb) * len(ks)), ndig, _pa([acc0]), _pa([acc1]), 0)

    cases = [
        ("k = 2", HB_ERR_INDEX_SET, lambda: call(ks=(1, 2))),
        ("k = 0", HB_ERR_INDEX_SET, lambda: call(ks=(1, 0))),
        ("k = m", HB_ERR_INDEX_SET, lambda: call(ks=(1, 64))),
        ("S with a special prime", HB_ERR_INDEX_SET, lambda: call(S_=Sbad)),
        ("seeded evk_a without a needed row", HB_ERR_INDEX_SET, lambda: call(ea=short)),
        ("ngiant = 0", HB_ERR_BAD_ARG, lambda: call(ngiant=0)),
        ("nbaby = 0", HB_ERR_BAD_ARG, lambda: call(nbaby=0)),
        ("nitems = 0", HB_ERR_BAD_ARG, lambda: call(nitems=0)),
        ("extended = 2", HB_ERR_BAD_ARG, lambda: call(ext=2)),
        ("ptxt_space = 0", HB_ERR_BAD_ARG, lambda: call(p=0)),
        ("too few matrix columns", HB_ERR_BAD_ARG, lambda: call(ndig=nd - 1)),
        ("scal != 1 in the extended form", HB_ERR_BAD_ARG, lambda: call(ext=1, scal=[1, 3])),
        ("acc0 = a baby step", HB_ERR_BAD_ARG, lambda: call(acc0=b0[0])),
        ("acc1 = a part-1 baby step", HB_ERR_BAD_ARG, lambda: call(acc1=b1[1])),
        ("acc0 = a constant", HB_ERR_BAD_ARG, lambda: call(acc0=cs[1])),
        ("acc1 = a matrix row", HB_ERR_BAD_ARG, lambda: call(acc1=EB[0])),
        ("acc0 = acc1", HB_ERR_BAD_ARG, lambda: call(acc1=a0)),
        ("seeded baby step", HB_ERR_BAD_ARG, lambda: call(B0=[Xs, b0[1]])),
        ("seeded constant", HB_ERR_BAD_ARG, lambda: call(consts=[Xs] + cs[1:] + cs)),
        ("seeded evk_b", HB_ERR_BAD_ARG, lambda: call(eb=[Xs] + EB[1:])),
        ("seeded acc0", HB_ERR_BAD_ARG, lambda: call(acc0=Xs)),
    ]
    assert call() == 0, L.hb_last_error()
    for name, code, f in cases:
        E.sync()
        before = E.stats()["launches"]
        rc = f()
        assert rc == code, (name, rc, L.hb_last_error())
        assert E.stats()["launches"] == before, name
    # a NULL constant is a zero diagonal, and an unrotated giant step needs no matrix
    assert call(consts=[None, cs[1], cs[0], None]) == 0, L.hb_last_error()
    kk = np.array([1], dtype=np.uint64)
    rc = L.hb_bsgs_linear_map(_pa(b0), _pa(b1), 2, 1, Sarr.ctypes.data_as(C.POINTER(C.c_int32)), len(Sarr), 0, C.c_uint64(257), 1,
                              kk.ctypes.data_as(C.POINTER(C.c_uint64)), _pa(cs), None, None, None, nd, _pa([a0]), _pa([a1]), 0)
    assert rc == 0, L.hb_last_error()
    E.close()


# ---- 4. code generation

def test_bsgs_kernels_keep_their_state_in_registers(engine_codegen):
    ptx, report = engine_codegen
    for name in ("k_bsgs_mac", "k_ks_giant"):
        frames = {k: v for k, v in _frames(report).items() if name in k}
        assert len(frames) == 3, (name, frames)
        assert all(v == (0, 0, 0) for v in frames.values()), frames
        assert not {k: v for k, v in _depots(ptx).items() if name in k}


# ---- 5. full size on the GPU: parity with the composed engine path, seeded keys, CUDA graph

def _full(cuda_lib, m, p, bits, c):
    from helib_b200 import Chain
    ch = Chain(m, p, 1, bits, c, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    return ch, E


def _full_case(E, ch, rng_seed, nb, ng, B, extended, gen):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    R = Sp if extended else S
    nd = len(ch.digits)
    ks = [pow(gen, (nb // (2 if extended else 1)) * t, ch.m) for t in range(ng)]
    B0 = [[E.poly() for _ in range(nb)] for _ in range(B)]
    B1 = [[E.poly() for _ in range(nb)] for _ in range(B)]
    E.randomize([x for it in B0 + B1 for x in it], R, rng_seed)
    CS = [[E.poly() for _ in range(nb)] for _ in range(ng)]
    E.randomize([x for row in CS for x in row], R, rng_seed + 1)
    CS[ng - 1][nb - 1] = None
    EB = [[E.poly() for _ in range(nd)] for _ in range(ng)]
    E.randomize([x for m_ in EB for x in m_], Sp, rng_seed + 2)
    EA = [[E.poly() for _ in range(nd)] for _ in range(ng)]
    for j, m_ in enumerate(EA):
        E.randomize(m_, Sp, rng_seed + 100 + j)
    SA = [E.seeded(nd, Sp, rng_seed + 100 + j) for j in range(ng)]
    return ks, B0, B1, CS, EA, EB, SA


@pytest.mark.gpu
@pytest.mark.parametrize("ring", ["cfg2", "cfg5"])
def test_full_size_matches_the_composed_engine_path(cuda_lib, ring):
    """Config 2's ring (CKKS m = 2^17, native form, 5 baby and 4 giant steps, relin_CKKS_adjust factors) and config 5's
    (m = 21845, p = 2, extended form, 2*3 baby and 3 giant steps): the fused call equals the composed engine path bit for bit,
    with expanded and with seeded matrices."""
    if ring == "cfg2":
        ch, E = _full(cuda_lib, 1 << 17, -1, 1190, 2)
        nb, ng, extended, p, scal = 5, 4, 0, 1, [1, 3, 1, 2]
    else:
        ch, E = _full(cuda_lib, 21845, 2, 580, 2)
        nb, ng, extended, p, scal = 6, 3, 1, 2, None
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    ks, B0, B1, CS, EA, EB, SA = _full_case(E, ch, 31, nb, ng, 3, extended, gen_of(ch.m))
    R0, R1 = [E.poly() for _ in range(3)], [E.poly() for _ in range(3)]
    composed(E, B0, B1, S, ks, CS, EA, EB, R0, R1, extended, p, scal)
    ref = [x.download(Sp)[Sp] for x in R0 + R1]
    for keys in (EA, SA):
        A0, A1 = [E.poly() for _ in range(3)], [E.poly() for _ in range(3)]
        E.bsgs_linear_map(B0, B1, S, ks, CS, keys, EB, A0, A1, extended=extended, ptxt_space=p, scal=scal)
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(ref, A0 + A1))
    E.close()


@pytest.mark.gpu
def test_config2_seeded_call_in_a_cuda_graph(cuda_lib):
    import torch
    ch, E = _full(cuda_lib, 1 << 17, -1, 1190, 2)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    ks, B0, B1, CS, EA, EB, SA = _full_case(E, ch, 41, 4, 5, 2, 0, gen_of(ch.m))
    A0, A1 = [E.poly() for _ in range(2)], [E.poly() for _ in range(2)]
    E.bsgs_linear_map(B0, B1, S, ks, CS, SA, EB, A0, A1)
    ref = [x.download(Sp)[Sp] for x in A0 + A1]
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    E.set_stream(side.cuda_stream)
    E.bsgs_linear_map(B0, B1, S, ks, CS, SA, EB, A0, A1)   # warm on the capturing stream
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        E.bsgs_linear_map(B0, B1, S, ks, CS, SA, EB, A0, A1)
    for _ in range(2):
        for x in A0 + A1:
            x.upload(np.zeros((E.np, E.N), dtype=np.uint64), Sp)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(ref, A0 + A1))
    torch.cuda.set_stream(torch.cuda.default_stream())
    E.close()


# ---- 6. the C++ mirror (tests/cpp/test_bsgs.cpp): hb::MatMul1DBSGS against the transcribed loop

def test_mirror_bsgs_on_simulator():
    r = subprocess.run([build_exe("test_bsgs", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "bsgs OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_bsgs_on_gpu():
    r = subprocess.run([build_exe("test_bsgs")], capture_output=True, text=True)
    assert r.returncode == 0 and "bsgs OK" in r.stdout, r.stdout + r.stderr
