"""Full linear map leaves (hb_full_linear_map_leaves, SURVEY 8f-1): the last dimension of MatMulFullExec::rec_mul
(src/matmul.cpp:2141-2148), every leaf a hoisted MatMul1DExec::mul (:1226-1283), all leaves of a ciphertext summed into one
accumulator.

Checked bit for bit against the oracle doing HElib's steps one by one (per leaf the cleanUp's mod-down, breakIntoDigits,
the hoisted rotations and MulAdd; for a bad leaf dimension the per-leaf second sum, then its automorph, mod-down,
breakIntoDigits, addPrimesAndScale and keySwitchDigits), against the existing entry points and the step-by-step engine
path at full size, with seeded matrices, at the largest primes, and for its argument errors.  Unless marked, each test
runs on the CPU simulator build and, marked gpu, on the H100.
"""
import ctypes as C
import subprocess

import numpy as np
import pytest

from bench_bsgs import gen_of
from bench_full_linear_map import WORKLOADS, existing_abi, leaf_amounts, step_by_step
from prg_sim import drop_stale_sim_build
from test_block_linear_map import _term
from test_bsgs import _ptxt, _rand, _setup
from test_codegen import _depots, _frames, engine_codegen  # noqa: F401  (module-scoped compile fixture)
from test_cpp_shim import build_exe
from test_value_ranges import all_minus_one_digits, bsgs_setup, const_rows, kernels, top

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
RINGS = [(64, 17, 1, 120, 2), (2048, 17, 2, 150, 3), (45, 2, 1, 100, 2), (105, 2, 1, 120, 2)]


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def _rot(X, ch, dig, c0, c1, k, ea, eb):
    """BasicAutomorphPrecon::automorph(k) of a cleaned ciphertext over S, over S | special."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    r0, r1 = c0.copy(), c1.copy()
    if k == 1:
        X.add_primes_and_scale(r0, S, ch.special)
        X.add_primes_and_scale(r1, S, ch.special)
        return r0, r1
    X.automorph(r0, S, k)
    X.add_primes_and_scale(r0, S, ch.special)
    r1 = X.zeros()
    rd = [d.copy() for d in dig]
    for d in rd:
        X.automorph(d, Sp, k)
    X.keyswitch_digits(rd, Sp, ea, eb, r0, r1)
    return r0, r1


def _reference(X, ch, x0s, x1s, ext, ks, ea, eb, cs, cs1, kf, eaf, ebf, acc0, acc1, rec=None):
    """The leaves of one ciphertext, step by step: per leaf cleanUp, breakIntoDigits, the hoisted rotations and MulAdd
    into the accumulator (and, bad, into the leaf's own second sum, then smartAutomorph(kf) of that sum).  rec (optional,
    a dict): per norm entry the polynomials whose norms hb_full_linear_map_leaves_norm reports."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    p = _ptxt(ch)
    acc0, acc1 = acc0.copy(), acc1.copy()
    nl = len(x0s)
    for l in range(nl):
        x0, x1 = x0s[l].copy(), x1s[l].copy()
        if rec is not None:
            rec[l] = {"moddown": (x0.copy(), x1.copy()) if ext[l] else None}
        if ext[l]:
            X.scale_down(x0, Sp, S, p)
            X.scale_down(x1, Sp, S, p)
        if rec is not None:
            rec[l]["part1"] = x1.copy()
        dig = X.break_into_digits(x1, S)
        y0, y1 = X.zeros(), X.zeros()
        for t, k in enumerate(ks):
            if cs[l][t] is None and (cs1 is None or cs1[l][t] is None):
                continue
            r0, r1 = _rot(X, ch, dig, x0, x1, k, ea[t], eb[t])
            if cs[l][t] is not None:
                X.muladd(acc0, r0, cs[l][t], Sp)
                X.muladd(acc1, r1, cs[l][t], Sp)
            if cs1 is not None and cs1[l][t] is not None:
                X.muladd(y0, r0, cs1[l][t], Sp)
                X.muladd(y1, r1, cs1[l][t], Sp)
        if cs1 is not None:
            got = []
            t0, t1 = _term(X, ch, y0, y1, kf, eaf, ebf, got)
            if rec is not None:
                rec[nl + l] = got
            X.add(acc0, t0, Sp)
            X.add(acc1, t1, Sp)
    return acc0, acc1


def _check(lib, cfg, ks, nleaves, bad=False, kf=None, nitems=2, ext=None, zero=(), zero_leaf=(), accumulate=False, seed=0,
           norms=False):
    """zero: (l, t) diagonals left None in both sets; zero_leaf: leaves whose diagonals are all None in both sets.
    norms: call hb_full_linear_map_leaves_norm and check every entry against hb_scale_down_norm / hb_break_into_digits_norm
    of the oracle's intermediate polynomials."""
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(seed)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N, na = len(ch.digits), E.N, len(ks)
    ext = [l % 3 != 0 for l in range(nleaves)] if ext is None else ext
    x0 = [[_rand(ch, rng, Sp if ext[l] else S, N) for l in range(nleaves)] for _ in range(nitems)]
    x1 = [[_rand(ch, rng, Sp if ext[l] else S, N) for l in range(nleaves)] for _ in range(nitems)]

    def diags():
        return [[None if (l, t) in zero or l in zero_leaf else _rand(ch, rng, Sp, N) for t in range(na)] for l in range(nleaves)]
    cs = diags()
    cs1 = diags() if bad else None

    def mats(kk):
        return [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) if k != 1 else None for k in kk]
    ea, eb = mats(ks), mats(ks)
    eaf, ebf = (mats([kf])[0], mats([kf])[0]) if bad else (None, None)
    a0 = [_rand(ch, rng, Sp, N) for _ in range(nitems)]
    a1 = [_rand(ch, rng, Sp, N) for _ in range(nitems)]

    def up(x):
        return E.poly(x, Sp) if x is not None else None

    def upm(ms):
        return [[E.poly(x, Sp) for x in m] if m is not None else None for m in ms]
    A0, A1 = [E.poly(x, Sp) for x in a0], [E.poly(x, Sp) for x in a1]
    X0 = [[E.poly(x, Sp if ext[l] else S) for l, x in enumerate(it)] for it in x0]
    X1 = [[E.poly(x, Sp if ext[l] else S) for l, x in enumerate(it)] for it in x1]
    got_norms = E.full_linear_map_leaves(X0, X1, S, ks, upm(ea), upm(eb), [[up(x) for x in r] for r in cs], A0, A1, ext=ext,
                                         consts1=[[up(x) for x in r] for r in cs1] if bad else None, kfinal=kf if bad else 1,
                                         evkf_a=upm([eaf])[0] if bad else None, evkf_b=upm([ebf])[0] if bad else None,
                                         ptxt_space=_ptxt(ch), accumulate=accumulate, norms=norms)
    for it in range(nitems):
        z = X.zeros()
        rec = {} if norms else None
        r0, r1 = _reference(X, ch, x0[it], x1[it], ext, ks, ea, eb, cs, cs1, kf, eaf, ebf,
                            a0[it] if accumulate else z, a1[it] if accumulate else z, rec)
        assert (A0[it].download(Sp)[Sp] == r0[Sp]).all() and (A1[it].download(Sp)[Sp] == r1[Sp]).all(), (cfg, it)
        for e, r in (rec or {}).items():
            if e < nleaves:
                _, dn = E.break_into_digits_norm([E.poly(r["part1"], S)], S)
                want = np.concatenate([dn[0], got_norms[it, e, len(dn[0]):8]])
                want = np.concatenate([want, E.scale_down_norm([E.poly(x, Sp) for x in r["moddown"]], Sp, S, _ptxt(ch))
                                       if r["moddown"] is not None else [np.nan, np.nan]])
            elif not r:   # kfinal == 1: the final term is not rotated, its entry is not written
                assert np.isnan(got_norms[it, e]).all(), (it, e)
                continue
            else:
                y0, y1 = E.poly(r[0][0], Sp), E.poly(r[0][1], Sp)
                sd = E.scale_down_norm([y0, y1], Sp, S, _ptxt(ch))
                _, dn = E.break_into_digits_norm([y1], S)
                want = np.concatenate([dn[0], got_norms[it, e, len(dn[0]):8], sd])
            assert np.allclose(got_norms[it, e], want, rtol=1e-9, atol=0, equal_nan=True), (cfg, it, e, got_norms[it, e], want)
    return E


def _dim(cfg, D):
    m = cfg[0]
    return leaf_amounts(m, gen_of(m), D)


# ---- 1. parity with the oracle

@pytest.mark.parametrize("shape", ["native", "bad"])
@pytest.mark.parametrize("cfg", RINGS)
def test_matches_helibs_steps(lib, cfg, shape):
    """5 leaves of 2 items, leaves 0 and 3 over S and the others over S | special; amount 0 is 1, one diagonal is NULL
    and leaf 2 has no diagonal at all."""
    ks, kf = _dim(cfg, 3)
    _check(lib, cfg, ks, 5, bad=shape == "bad", kf=kf, zero={(1, 1)}, zero_leaf={2}, seed=cfg[0] + len(shape)).close()


@pytest.mark.parametrize("cfg", [(64, 17, 1, 120, 2), (105, 2, 1, 120, 2)])
def test_accumulate_and_every_leaf_over_s(lib, cfg):
    ks, kf = _dim(cfg, 3)
    _check(lib, cfg, ks, 3, bad=True, kf=kf, ext=[0, 0, 0], accumulate=True, seed=9).close()
    _check(lib, cfg, ks, 3, bad=False, ext=[1, 1, 1], accumulate=True, seed=10).close()


def test_leaf_and_amount_chunks(lib):
    """37 leaves of 1 item and 40 amounts: two leaf chunks of 32 and 5 (the second with a k_ks_leafmap<4> group and a
    one-leaf tail), two amount groups of 32 and 8, and 32 x 32 = 1024 terms, more than the 255 a 128-bit sum holds, in
    the accumulators of the first launch."""
    cfg = (64, 17, 1, 120, 2)
    ks = [pow(3, i, 64) for i in range(40)]
    _check(lib, cfg, ks, 37, nitems=1, seed=37).close()
    _check(lib, cfg, ks, 37, nitems=1, bad=True, kf=pow(3, -40, 64), accumulate=True, seed=38).close()


def test_item_chunks(lib):
    """9 items of 6 leaves: chunks of 8 items x 4 leaves (at most 32 pairs), so two item chunks (8 + 1) and two leaf chunks
    (4 + 2, the second k_ks_leafmap<2>); 2 items of 3 leaves: k_ks_leafmap<2> and a one-leaf tail."""
    cfg = (64, 17, 1, 120, 2)
    ks, kf = _dim(cfg, 3)
    _check(lib, cfg, ks, 6, nitems=9, bad=True, kf=kf, seed=6).close()
    _check(lib, cfg, ks, 3, nitems=2, seed=7).close()


def test_final_amount_one(lib):
    cfg = (45, 2, 1, 100, 2)
    ks, _ = _dim(cfg, 2)
    _check(lib, cfg, ks, 3, bad=True, kf=1, seed=1, norms=True).close()


# ---- norms (hb_full_linear_map_leaves_norm)

def test_norms_native(lib):
    cfg = (64, 17, 1, 120, 2)
    ks, _ = _dim(cfg, 3)
    _check(lib, cfg, ks, 5, nitems=2, zero_leaf={2}, norms=True, seed=81).close()


def test_norms_bad_across_chunks(lib):
    """9 items of 6 leaves: chunks of 8 items x 4 leaves, so the second item chunk starts at item 8 and every leaf chunk but
    the first at leaf 4; the final terms' entries follow the leaf entries."""
    cfg = (64, 17, 1, 120, 2)
    ks, kf = _dim(cfg, 3)
    _check(lib, cfg, ks, 6, nitems=9, bad=True, kf=kf, norms=True, seed=82).close()


def test_norms_general_m(lib):
    cfg = (105, 2, 1, 120, 2)
    ks, kf = _dim(cfg, 3)
    _check(lib, cfg, ks, 4, nitems=2, bad=True, kf=kf, norms=True, seed=84).close()


# ---- 2. worst case at the largest primes

@pytest.mark.parametrize("m", [64, 105])
def test_sums_at_q_minus_one(lib, m):
    """Every reduced inner product and every constant is q-1 (so each term of the accumulators' 128-bit sums is (q-1)^2,
    the largest product of reduced values), on chains of the largest primes below 2^60: leaves over S whose part 1 is the
    constant with all-(-1) digits, part 0 and the accumulators at q-1, and keys a_0 = nd, b_0 = nd - P, every other key
    q-1.  33 leaves x 40 amounts of one item: 32 x 32 = 1024 terms in the first launch's sums, against the budget
    "reduced and carried before it holds 255 terms (its old value counts as one)" of k_ks_leafmap (hb_device.cuh); the
    bad dimension's per-leaf sums hold HB_LEAF_MAXAMT + 1 terms."""
    nd = 3
    ch, X, E = bsgs_setup(lib, m, nd)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    P = ch.product(ch.special)
    ea = np.stack([top(ch, Sp) for _ in range(nd)])
    eb = ea.copy()
    for r in Sp:
        q = ch.primes[r]
        ea[0][r] = nd % q
        eb[0][r] = (nd - (P if r in S else 0)) % q
    u = [t for t in range(2, m) if np.gcd(t, m) == 1]
    ks = [u[j % len(u)] for j in range(40)]
    kf = u[1]
    nl = 33
    x0, x1 = top(ch, S), const_rows(ch, S, all_minus_one_digits(ch, S))
    cst = top(ch, Sp)
    EA = [E.poly(ea[i], Sp) for i in range(nd)]
    EB = [E.poly(eb[i], Sp) for i in range(nd)]
    CS = E.poly(cst, Sp)
    X0, X1 = [[E.poly(x0, S) for _ in range(nl)]], [[E.poly(x1, S) for _ in range(nl)]]
    for bad in (False, True):
        A0, A1 = [E.poly(top(ch, Sp), Sp)], [E.poly(top(ch, Sp), Sp)]
        E.profile(True)
        E.full_linear_map_leaves(X0, X1, S, ks, [EA] * len(ks), [EB] * len(ks), [[CS] * len(ks)] * nl, A0, A1, ext=[0] * nl,
                                 consts1=[[CS] * len(ks)] * nl if bad else None, kfinal=kf, evkf_a=EA if bad else None,
                                 evkf_b=EB if bad else None, ptxt_space=_ptxt(ch), accumulate=True)
        E.profile(False)
        assert "k_ks_leafmap" in kernels(E), kernels(E)
        # the construction: every reduced inner product is -1
        dig = X.break_into_digits(x1.copy(), S)
        r0, r1 = _rot(X, ch, dig, x0, x1, ks[0], ea, eb)
        assert all((r0[r] == ch.primes[r] - 1).all() and (r1[r] == ch.primes[r] - 1).all() for r in Sp)
        acc = top(ch, Sp)
        w0, w1 = _reference(X, ch, [x0] * nl, [x1] * nl, [0] * nl, ks, [ea] * len(ks), [eb] * len(ks),
                            [[cst] * len(ks)] * nl, [[cst] * len(ks)] * nl if bad else None, kf, ea, eb, acc, acc)
        assert (A0[0].download(Sp)[Sp] == w0[Sp]).all() and (A1[0].download(Sp)[Sp] == w1[Sp]).all(), bad
    E.close()


# ---- 3. seeded matrices, scratch

def _case(E, ch, rng, nl, na, nitems, bad):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    ks = [pow(gen_of(ch.m), i, ch.m) for i in range(na)]
    ext = [l % 2 for l in range(nl)]
    X0 = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nl)] for _ in range(nitems)]
    X1 = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nl)] for _ in range(nitems)]
    CS = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(na)] for _ in range(nl)]
    CS1 = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(na)] for _ in range(nl)] if bad else None
    EB = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(na)]
    return ks, ext, X0, X1, CS, CS1, EB


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (105, 2, 1, 120, 2)])
def test_seeded_expanded_and_mixed_matrices_agree(lib, cfg):
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(5)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    ks, ext, X0, X1, CS, CS1, EB = _case(E, ch, rng, 6, 5, 2, True)
    EBf = [E.poly(_rand(ch, rng, Sp, E.N), Sp) for _ in range(nd)]

    def keys(n, seed):
        s = [E.seeded(nd, Sp, seed + j) for j in range(n)]
        x = []
        for j in range(n):
            P_ = [E.poly() for _ in range(nd)]
            E.randomize(P_, Sp, seed + j)
            x.append(P_)
        return x, s, [s[j] if j % 2 else x[j] for j in range(n)]
    K, Kf = keys(5, 100), keys(1, 300)
    outs = []
    for f in range(3):
        A0, A1 = [E.poly() for _ in X0], [E.poly() for _ in X0]
        E.full_linear_map_leaves(X0, X1, S, ks, [None if k == 1 else m_ for k, m_ in zip(ks, K[f])], EB, CS, A0, A1, ext=ext,
                                 consts1=CS1, kfinal=ks[1], evkf_a=Kf[f][0], evkf_b=EBf, ptxt_space=_ptxt(ch))
        outs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[1]))
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[2]))
    E.close()


def test_scratch_does_not_grow_with_the_leaves(sim_lib):
    """One item of 32 leaves and 40 amounts with seeded matrices fills the leaf scratch (a whole chunk, bad dimension,
    seeded final matrix) and the key scratch; 96 leaves then need nothing more."""
    ch, X, E = _setup(sim_lib, (64, 17, 1, 120, 2))
    rng = np.random.default_rng(6)
    Sp = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    ks, ext, X0, X1, CS, CS1, EB = _case(E, ch, rng, 96, 4, 1, True)
    SA = [E.seeded(nd, Sp, 77 + j) for j in range(4)]
    SAf = E.seeded(nd, Sp, 7)
    A0, A1 = [E.poly()], [E.poly()]
    pick = [1 + j % 3 for j in range(40)]

    def run(nl):
        E.full_linear_map_leaves([X0[0][:nl]], [X1[0][:nl]], ch.ctxt, [ks[j] for j in pick], [SA[j] for j in pick],
                                 [EB[j] for j in pick], [[r[j] for j in pick] for r in CS[:nl]], A0, A1, ext=ext[:nl],
                                 consts1=[[r[j] for j in pick] for r in CS1[:nl]], kfinal=ks[1], evkf_a=SAf, evkf_b=EB[1],
                                 ptxt_space=17)
    run(32)
    first = E.stats()["device_bytes"]
    run(96)
    assert E.stats()["device_bytes"] == first
    E.close()


# ---- 4. argument errors: each reported before any launch

_KEEP = []


def _pa(lst):
    a = (C.c_void_p * max(1, len(lst)))(*[None if p is None else p.h for p in lst])
    _KEEP.append(a)
    return a


def _np(xs, dt, ct):
    a = np.ascontiguousarray(np.array(xs, dtype=dt))
    _KEEP.append(a)
    return a.ctypes.data_as(C.POINTER(ct))


def test_argument_errors_launch_nothing(sim_lib):
    ch, X, E = _setup(sim_lib, (64, 17, 1, 120, 2))
    rng = np.random.default_rng(8)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    L = E.lib
    x0 = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(2)]
    x1 = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(2)]
    cs = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(4)]
    EA = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    EB = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    a0, a1 = E.poly(), E.poly()
    Xs = E.seeded(1, Sp, 5)[0]
    short = E.seeded(nd, sorted(ch.ctxt[:-1] + ch.special), 6)    # lacks the top ctxt prime
    Sarr = np.ascontiguousarray(np.array(S, dtype=np.int32))
    Sbad = np.ascontiguousarray(np.array(S + ch.special[:1], dtype=np.int32))

    def call(X0=x0, X1=x1, nl=2, nitems=1, ext=(0, 1), S_=Sarr, p=17, ks=(1, 3), ea=EA, eb=EB, consts=None, consts1=False,
             kf=5, eaf=EA, ndig=nd, acc0=a0, acc1=a1, na=None):
        consts = consts if consts is not None else cs
        c1s = (cs if consts1 is False else consts1) if consts1 is not None else None
        return L.hb_full_linear_map_leaves(_pa(X0), _pa(X1), nl, nitems, _np(ext, np.int32, C.c_int32) if ext is not None else None,
                                           S_.ctypes.data_as(C.POINTER(C.c_int32)), len(S_), C.c_uint64(p),
                                           len(ks) if na is None else na, _np(ks, np.uint64, C.c_uint64),
                                           _pa(list(ea) * len(ks)), _pa(list(eb) * len(ks)), _pa(consts),
                                           _pa(c1s) if c1s is not None else None, C.c_uint64(kf), _pa(eaf), _pa(EB), ndig,
                                           _pa([acc0]), _pa([acc1]), 0)

    cases = [
        ("k = 2", HB_ERR_INDEX_SET, lambda: call(ks=(1, 2))),
        ("k = 0", HB_ERR_INDEX_SET, lambda: call(ks=(0, 3))),
        ("k = m", HB_ERR_INDEX_SET, lambda: call(ks=(1, 64))),
        ("kfinal = 4", HB_ERR_INDEX_SET, lambda: call(kf=4)),
        ("S with a special prime", HB_ERR_INDEX_SET, lambda: call(S_=Sbad)),
        ("seeded evk_a without a needed row", HB_ERR_INDEX_SET, lambda: call(ea=short)),
        ("seeded evkf_a without a needed row", HB_ERR_INDEX_SET, lambda: call(eaf=short)),
        ("nleaves = 0", HB_ERR_BAD_ARG, lambda: call(nl=0)),
        ("namt = 0", HB_ERR_BAD_ARG, lambda: call(na=0)),
        ("nitems = 0", HB_ERR_BAD_ARG, lambda: call(nitems=0)),
        ("ext = 2", HB_ERR_BAD_ARG, lambda: call(ext=(0, 2))),
        ("ptxt_space = 0", HB_ERR_BAD_ARG, lambda: call(p=0)),
        ("too few matrix columns", HB_ERR_BAD_ARG, lambda: call(ndig=nd - 1)),
        ("missing matrix", HB_ERR_BAD_ARG, lambda: call(ea=[None] * nd)),
        ("acc0 = a leaf part", HB_ERR_BAD_ARG, lambda: call(acc0=x0[1])),
        ("acc1 = a constant", HB_ERR_BAD_ARG, lambda: call(acc1=cs[2])),
        ("acc0 = a matrix row", HB_ERR_BAD_ARG, lambda: call(acc0=EB[0])),
        ("acc0 = acc1", HB_ERR_BAD_ARG, lambda: call(acc1=a0)),
        ("seeded leaf", HB_ERR_BAD_ARG, lambda: call(X1=[x1[0], Xs])),
        ("seeded constant", HB_ERR_BAD_ARG, lambda: call(consts=[Xs] + cs[1:])),
        ("seeded set-1 constant", HB_ERR_BAD_ARG, lambda: call(consts1=cs[:3] + [Xs])),
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
    # NULL constants are zero diagonals, every leaf over S needs no ext, and a native call needs no final amount
    assert call(consts=[None, cs[1], None, None], consts1=None, kf=4, ext=None) == 0, L.hb_last_error()
    E.close()


# ---- 5. code generation

def test_leaf_kernel_keeps_its_state_in_registers(engine_codegen):
    ptx, report = engine_codegen
    frames = {k: v for k, v in _frames(report).items() if "k_ks_leafmap" in k}
    assert len(frames) == 6, frames
    assert all(v == (0, 0, 0) for v in frames.values()), frames
    assert not {k: v for k, v in _depots(ptx).items() if "k_ks_leafmap" in k}


# ---- 6. full size on the GPU: parity with the existing entry points and the step-by-step path

@pytest.mark.gpu
@pytest.mark.parametrize("key", ["cfg5", "cfg3"])
def test_full_size_matches_the_engine_paths(cuda_lib, key):
    """Config 5's ring (m = 21845, p = 2) with its leaf dimension (bad, generator 21591, D = 16) under the 4 x 16 outer
    dimensions, and config 3's (m = 2^17, p = 257) with 16 x 16 synthetic native dimensions, 2 ciphertexts: the fused call,
    with expanded and with seeded matrices, equals one existing call per leaf and the step-by-step engine path bit for
    bit, and the launch profile shows k_ks_leafmap ran."""
    from helib_b200 import Chain
    from helib_b200.engine import Engine
    m, p, bits, c = {"cfg5": (21845, 2, 580, 2), "cfg3": (1 << 17, 257, 1500, 3)}[key]
    _, nl, gen, D, bad = WORKLOADS[key]
    if key == "cfg3":
        nl = 8   # a shorter outer dimension keeps the test's memory small (one chunk of 2 items x 8 leaves)
    ch = Chain(m, p, 1, bits, c, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, B = len(ch.digits), 2
    ks, kf = leaf_amounts(m, gen, D)
    ext = [0] + [1] * (nl - 1)
    X0 = [[E.poly() for _ in range(nl)] for _ in range(B)]
    X1 = [[E.poly() for _ in range(nl)] for _ in range(B)]
    E.randomize([x for it in X0 + X1 for x in it], Sp, 11)
    CS = [[E.poly() for _ in ks] for _ in range(nl)]
    CS1 = [[E.poly() for _ in ks] for _ in range(nl)] if bad else None
    E.randomize([x for r in CS + (CS1 or []) for x in r], Sp, 12)
    CS[nl - 1][3] = None

    def mats(kk, seed):
        EA = [None if k == 1 else [E.poly() for _ in range(nd)] for k in kk]
        EB = [None if k == 1 else [E.poly() for _ in range(nd)] for k in kk]
        SA = [None if k == 1 else E.seeded(nd, Sp, seed + j) for j, k in enumerate(kk)]
        for j, k in enumerate(kk):
            if k != 1:
                E.randomize(EA[j], Sp, seed + j)
                E.randomize(EB[j], Sp, seed + 500 + j)
        return EA, EB, SA
    EA, EB, SA = mats(ks, 1000)
    EAf, EBf, SAf = mats([kf], 3000) if bad else ([None], [None], [None])
    one = E.poly(np.ones((E.np, E.N), dtype=np.uint64), Sp)
    W0, W1, Y0, Y1, Z0, Z1 = ([E.poly() for _ in range(B)] for _ in range(6))
    DG = [[E.poly() for _ in range(nd)] for _ in range(B)]
    R0 = [[E.poly() for _ in ks] for _ in range(B)]
    R1 = [[E.poly() for _ in ks] for _ in range(B)]
    tmp = [[E.poly() for _ in range(B)] for _ in range(5)]
    extra = dict(cs1=CS1, kf=kf, EAf=EAf[0], EBf=EBf[0]) if bad else {}
    refs = []
    for route in (existing_abi, step_by_step):
        A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        kw = dict(R0=R0, R1=R1, Y0=Y0, Y1=Y1, Z0=Z0, Z1=Z1, one=one, tmp=tmp) if route is step_by_step else {}
        route(E, X0, X1, ext, S, ks, EA, EB, CS, A0, A1, p, W0=W0, W1=W1, DG=DG, **extra, **kw)
        refs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(refs[0], refs[1]))
    for ka, kaf in ((EA, EAf), (SA, SAf)):
        A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        E.profile(True)
        E.full_linear_map_leaves(X0, X1, S, ks, ka, EB, CS, A0, A1, ext=ext, consts1=CS1, kfinal=kf, evkf_a=kaf[0],
                                 evkf_b=EBf[0], ptxt_space=p)
        E.profile(False)
        assert "k_ks_leafmap" in kernels(E), kernels(E)
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(refs[0], A0 + A1))
    E.close()


# ---- 7. the C++ mirror (tests/cpp/test_matmul_full.cpp): hb::MatMulFull and hb::MatMul1D against the transcribed loops

def test_mirror_matmul_full_on_simulator():
    r = subprocess.run([build_exe("test_matmul_full", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "matmul full OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_matmul_full_on_gpu():
    r = subprocess.run([build_exe("test_matmul_full")], capture_output=True, text=True)
    assert r.returncode == 0 and "matmul full OK" in r.stdout, r.stdout + r.stderr
