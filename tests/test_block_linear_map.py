"""Block linear maps (hb_block_linear_map, SURVEY 8f-1): BlockMatMul1DExec::mul's non-iterative branches with one
interval (src/matmul.cpp:1782-1868 native, 1869-1974 bad dimension).

Checked bit for bit against the oracle doing HElib's steps one by one (the hoisted rotations, MulAdd of every block, then
per outer amount automorph, the mod-down of reLinearize, breakIntoDigits, addPrimesAndScale and keySwitchDigits, and the
adds; in a bad dimension the same for the second set and the final rotation), against the existing entry points and the
step-by-step engine path at full size, with seeded matrices, and for its argument errors.  Unless marked, each test runs
on the CPU simulator build and, marked gpu, on the H100.
"""
import ctypes as C
import subprocess

import numpy as np
import pytest

from bench_block_linear_map import amounts, existing_abi, step_by_step
from bench_bsgs import gen_of
from helib_b200.engine import Engine
from prg_sim import drop_stale_sim_build
from test_bsgs import _ptxt, _rand, _setup
from test_codegen import _depots, _frames, engine_codegen  # noqa: F401  (module-scoped compile fixture)
from test_cpp_shim import build_exe

drop_stale_sim_build()

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
RINGS = [(64, 17, 1, 120, 2), (2048, 17, 2, 150, 3), (45, 2, 1, 100, 2), (105, 2, 1, 120, 2), (1285, 2, 1, 120, 2)]


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def _term(X, ch, x0, x1, k, ea, eb, rec=None):
    """smartAutomorph(k) of an extended ciphertext over S | special: automorph, mod-down, breakIntoDigits, key switch.
    rec (optional): receives the rotated sum before its mod-down."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    x0, x1 = x0.copy(), x1.copy()
    if k == 1:
        return x0, x1
    X.automorph(x0, Sp, k)
    X.automorph(x1, Sp, k)
    if rec is not None:
        rec.append((x0.copy(), x1.copy()))
    X.scale_down(x0, Sp, S, _ptxt(ch))
    X.scale_down(x1, Sp, S, _ptxt(ch))
    digs = X.break_into_digits(x1, S)
    r0, r1 = x0.copy(), X.zeros()
    X.add_primes_and_scale(r0, S, ch.special)
    X.keyswitch_digits(digs, Sp, ea, eb, r0, r1)
    return r0, r1


def _reference(X, ch, dig, c0, c1, k0, ea0, eb0, k1, ea1, eb1, cs, cs1, kf, eaf, ebf, acc0, acc1, rec=None):
    """BlockMatMul1DExec::mul's loop, step by step: the hoisted rotations, MulAdd into d1 sums per set, then the outer
    rotations summed (and the set-1 sum rotated by kf).  rec (optional, a dict): the rotated sum of every rotated term
    before its mod-down, under its entry in hb_block_linear_map_norm's layout."""
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    rot = []
    for i, k in enumerate(k0):
        r0, r1 = c0.copy(), c1.copy()
        if k == 1:
            X.add_primes_and_scale(r0, S, ch.special)
            X.add_primes_and_scale(r1, S, ch.special)
        else:
            X.automorph(r0, S, k)
            X.add_primes_and_scale(r0, S, ch.special)
            r1 = X.zeros()
            rd = [d.copy() for d in dig]
            for d in rd:
                X.automorph(d, Sp, k)
            X.keyswitch_digits(rd, Sp, ea0[i], eb0[i], r0, r1)
        rot.append((r0, r1))

    n1 = len(k1)

    def entry(e):
        got = []
        if rec is not None:
            rec[e] = got
        return got

    def half(blocks, set_):
        s0, s1 = X.zeros(), X.zeros()
        for j, k in enumerate(k1):
            a0, a1 = X.zeros(), X.zeros()
            for i, (r0, r1) in enumerate(rot):
                if blocks[i][j] is not None:
                    X.muladd(a0, r0, blocks[i][j], Sp)
                    X.muladd(a1, r1, blocks[i][j], Sp)
            t0, t1 = _term(X, ch, a0, a1, k, ea1[j], eb1[j], entry(set_ * n1 + j))
            X.add(s0, t0, Sp)
            X.add(s1, t1, Sp)
        return s0, s1

    acc0, acc1 = acc0.copy(), acc1.copy()
    s0, s1 = half(cs, 0)
    X.add(acc0, s0, Sp)
    X.add(acc1, s1, Sp)
    if cs1 is not None:
        y0, y1 = half(cs1, 1)
        t0, t1 = _term(X, ch, y0, y1, kf, eaf, ebf, entry(2 * n1))
        X.add(acc0, t0, Sp)
        X.add(acc1, t1, Sp)
    return acc0, acc1


def _check(lib, cfg, k0, k1, bad=False, kf=None, nitems=2, zero=(), zero_out=(), accumulate=False, seed=0, norms=False):
    """zero: (i, j) blocks left None in both sets; zero_out: outer amounts j whose blocks are all None in set 0.
    norms: call hb_block_linear_map_norm and check every entry against the digit and mod-down norms that the single-step
    entry points (hb_scale_down_norm, hb_break_into_digits_norm) give the oracle's rotated sums."""
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(seed)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N, n0, n1 = len(ch.digits), E.N, len(k0), len(k1)
    dig = [[_rand(ch, rng, Sp, N) for _ in range(nd)] for _ in range(nitems)]
    c0 = [_rand(ch, rng, S, N) for _ in range(nitems)]
    c1 = [_rand(ch, rng, S, N) for _ in range(nitems)]

    def blocks(skip_out):
        return [[None if (i, j) in zero or j in skip_out else _rand(ch, rng, Sp, N) for j in range(n1)] for i in range(n0)]
    cs = blocks(zero_out)
    cs1 = blocks(()) if bad else None

    def mats(ks):
        return [np.stack([_rand(ch, rng, Sp, N) for _ in range(nd)]) if k != 1 else None for k in ks]
    ea0, eb0, ea1, eb1 = mats(k0), mats(k0), mats(k1), mats(k1)
    eaf, ebf = (mats([kf])[0], mats([kf])[0]) if bad else (None, None)
    a0 = [_rand(ch, rng, Sp, N) for _ in range(nitems)]
    a1 = [_rand(ch, rng, Sp, N) for _ in range(nitems)]

    def up(x, idx):
        return E.poly(x, idx) if x is not None else None

    def upm(ms):
        return [[E.poly(x, Sp) for x in m] if m is not None else None for m in ms]
    A0, A1 = [E.poly(x, Sp) for x in a0], [E.poly(x, Sp) for x in a1]   # overwritten when not accumulating
    got_norms = E.block_linear_map([[E.poly(x, Sp) for x in d] for d in dig], S, [E.poly(x, S) for x in c0], [E.poly(x, S) for x in c1],
                       k0, upm(ea0), upm(eb0), k1, upm(ea1), upm(eb1), [[up(x, Sp) for x in r] for r in cs], A0, A1,
                       consts1=[[up(x, Sp) for x in r] for r in cs1] if bad else None, kfinal=kf if bad else 1,
                       evkf_a=upm([eaf])[0] if bad else None, evkf_b=upm([ebf])[0] if bad else None,
                       ptxt_space=_ptxt(ch), accumulate=accumulate, norms=norms)
    for it in range(nitems):
        z = X.zeros()
        rec = {} if norms else None
        r0, r1 = _reference(X, ch, dig[it], c0[it], c1[it], k0, ea0, eb0, k1, ea1, eb1, cs, cs1, kf, eaf, ebf,
                            a0[it] if accumulate else z, a1[it] if accumulate else z, rec)
        assert (A0[it].download(Sp)[Sp] == r0[Sp]).all() and (A1[it].download(Sp)[Sp] == r1[Sp]).all(), (cfg, it)
        for e, got in (rec or {}).items():
            if not got:   # an unrotated term: its entry is not written
                assert np.isnan(got_norms[it, e]).all(), (it, e)
                continue
            x0, x1 = E.poly(got[0][0], Sp), E.poly(got[0][1], Sp)
            sd = E.scale_down_norm([x0, x1], Sp, S, _ptxt(ch))
            _, dn = E.break_into_digits_norm([x1], S)
            want = np.concatenate([dn[0], got_norms[it, e, len(dn[0]):8], sd])
            assert np.allclose(got_norms[it, e], want, rtol=1e-9, atol=0, equal_nan=True), (cfg, it, e, got_norms[it, e], want)
    E.close()


def _dim(cfg, D, d):
    """A dimension of order D over slots of degree d: BlockMatMul1DExec's amounts for the ring's generator and p."""
    m, p = cfg[0], cfg[1]
    return amounts(m, p, gen_of(m), D, d)


# ---- 1. parity with the oracle

@pytest.mark.parametrize("shape", ["plus-native", "minus-native", "plus-bad", "minus-bad"])
@pytest.mark.parametrize("cfg", RINGS)
def test_matches_helibs_steps(lib, cfg, shape):
    """Strategy +1 (D >= d: the dimension hoisted, the Frobenius outside) and -1, native and bad; k0 = 1 is amount 0, one
    block is NULL and set 0's outer amount 1 has no block at all."""
    D, d = (3, 2) if shape.startswith("plus") else (2, 3)
    k0, k1, kf = _dim(cfg, D, d)
    _check(lib, cfg, k0, k1, bad=shape.endswith("bad"), kf=kf, zero={(0, 0)}, zero_out={1}, seed=cfg[0] + len(shape))


@pytest.mark.parametrize("cfg", [(64, 17, 1, 120, 2), (105, 2, 1, 120, 2)])
def test_repeated_amount_and_accumulate(lib, cfg):
    k0, k1, kf = _dim(cfg, 3, 2)
    _check(lib, cfg, k0 + [k0[1]], k1, bad=True, kf=kf, accumulate=True, seed=9)


def test_more_than_64_inner_amounts(lib):
    """70 inner amounts: two k_ks_hoist launches in one chunk (1 item), and two chunks per group (3 items)."""
    cfg = (64, 17, 1, 120, 2)
    k0 = [pow(3, i, 64) for i in range(70)]
    _check(lib, cfg, k0, [1, 17], nitems=1, seed=70)
    _check(lib, cfg, k0, [1, 17], nitems=3, bad=True, kf=pow(3, -16, 64), accumulate=True, seed=71)


def test_outputs_across_groups(lib):
    """12 outer amounts in both sets of 3 items: 72 (output, item) pairs, more than one group of 64."""
    cfg = (64, 17, 1, 120, 2)
    k1 = [pow(3, j, 64) for j in range(12)]
    _check(lib, cfg, [1, 17], k1, nitems=3, bad=True, kf=pow(3, -12, 64), seed=12)


@pytest.mark.parametrize("cfg", [(64, 17, 1, 120, 2), (45, 2, 1, 100, 2)])
def test_four_items_per_thread(lib, cfg):
    """5 items: k_ks_hoist<4> and its one-item tail in the second item group."""
    k0, k1, kf = _dim(cfg, 3, 2)
    _check(lib, cfg, k0, k1, bad=True, kf=kf, nitems=5, zero={(1, 0)}, seed=5)


# ---- norms (hb_block_linear_map_norm): every rotated term's entry, where the call's groups and item chunks split

def test_norms_native(lib):
    cfg = (64, 17, 1, 120, 2)
    k0, k1, _ = _dim(cfg, 3, 2)
    _check(lib, cfg, k0, k1, nitems=2, zero_out={1}, norms=True, seed=81)


def test_norms_bad_dimension_across_groups(lib):
    """3 items, 12 outer amounts in both sets: set 1's outputs straddle the first and second group of 64 pairs."""
    cfg = (64, 17, 1, 120, 2)
    k1 = [pow(3, j, 64) for j in range(12)]
    _check(lib, cfg, [1, 17], k1, nitems=3, bad=True, kf=pow(3, -12, 64), norms=True, seed=82)


def test_norms_across_item_chunks(lib):
    """33 items: two item chunks of at most 32."""
    cfg = (64, 17, 1, 120, 2)
    _check(lib, cfg, [1, 17], [1, 3], nitems=33, bad=True, kf=pow(3, -2, 64), norms=True, seed=83)


def test_norms_general_m(lib):
    cfg = (105, 2, 1, 120, 2)
    k0, k1, kf = _dim(cfg, 3, 2)
    _check(lib, cfg, k0, k1, bad=True, kf=kf, nitems=2, norms=True, seed=84)


def test_final_amount_one(lib):
    cfg = (45, 2, 1, 100, 2)
    k0, k1, _ = _dim(cfg, 2, 2)
    _check(lib, cfg, k0, k1, bad=True, kf=1, seed=1)


# ---- 2. seeded matrices, scratch

def _case(E, ch, rng, n0, n1, nitems):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    k0 = [pow(gen_of(ch.m), i, ch.m) for i in range(n0)]
    k1 = [pow(ch.p, j, ch.m) for j in range(n1)]
    D = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(nitems)]
    C0 = [E.poly(_rand(ch, rng, S, N), S) for _ in range(nitems)]
    C1 = [E.poly(_rand(ch, rng, S, N), S) for _ in range(nitems)]
    CS = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(n1)] for _ in range(n0)]
    EB0 = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(n0)]
    EB1 = [[E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)] for _ in range(n1)]
    return k0, k1, D, C0, C1, CS, EB0, EB1


@pytest.mark.parametrize("cfg", [(2048, 17, 2, 150, 3), (105, 2, 1, 120, 2)])
def test_seeded_expanded_and_mixed_matrices_agree(lib, cfg):
    ch, X, E = _setup(lib, cfg)
    rng = np.random.default_rng(5)
    Sp = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    k0, k1, D, C0, C1, CS, EB0, EB1 = _case(E, ch, rng, 5, 3, 2)
    EBf = [E.poly(_rand(ch, rng, Sp, E.N), Sp) for _ in range(nd)]

    def keys(n, seed):
        s = [E.seeded(nd, Sp, seed + j) for j in range(n)]
        x = []
        for j in range(n):
            P = [E.poly() for _ in range(nd)]
            E.randomize(P, Sp, seed + j)
            x.append(P)
        return x, s, [s[j] if j % 2 else x[j] for j in range(n)]
    K0, K1, Kf = keys(5, 100), keys(3, 200), keys(1, 300)
    outs = []
    for f in range(3):
        A0, A1 = [E.poly() for _ in D], [E.poly() for _ in D]
        E.block_linear_map(D, ch.ctxt, C0, C1, k0, K0[f], EB0, k1, K1[f], EB1, CS, A0, A1, consts1=CS, kfinal=k0[1],
                           evkf_a=Kf[f][0], evkf_b=EBf, ptxt_space=_ptxt(ch))
        outs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[1]))
    assert all(np.array_equal(a, b) for a, b in zip(outs[0], outs[2]))
    E.close()


def test_scratch_does_not_grow_with_the_inner_amounts(sim_lib):
    """16 items fill the rotation scratch at 8 inner amounts (none of them 1, so each regeneration of seeded matrices is
    full too); 64 then need nothing more."""
    ch, X, E = _setup(sim_lib, (64, 17, 1, 120, 2))
    rng = np.random.default_rng(6)
    Sp = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    k0, k1, D, C0, C1, CS, EB0, EB1 = _case(E, ch, rng, 64, 2, 16)
    SA0 = [E.seeded(nd, Sp, 77 + j) for j in range(64)]
    SA1 = [E.seeded(nd, Sp, 7 + j) for j in range(2)]
    A0, A1 = [E.poly() for _ in D], [E.poly() for _ in D]
    E.block_linear_map(D, ch.ctxt, C0, C1, k0[1:9], SA0[1:9], EB0[1:9], k1, SA1, EB1, CS[1:9], A0, A1, ptxt_space=17)
    eight = E.stats()["device_bytes"]
    E.block_linear_map(D, ch.ctxt, C0, C1, k0, SA0, EB0, k1, SA1, EB1, CS, A0, A1, ptxt_space=17)
    assert E.stats()["device_bytes"] == eight
    E.close()


# ---- 3. argument errors: each reported before any launch

_KEEP = []


def _pa(lst):
    a = (C.c_void_p * max(1, len(lst)))(*[None if p is None else p.h for p in lst])
    _KEEP.append(a)
    return a


def _u64(xs):
    a = np.ascontiguousarray(np.array(xs, dtype=np.uint64))
    _KEEP.append(a)
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def test_argument_errors_launch_nothing(sim_lib):
    ch, X, E = _setup(sim_lib, (64, 17, 1, 120, 2))
    rng = np.random.default_rng(8)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, N = len(ch.digits), E.N
    L = E.lib
    dg = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    c0, c1 = E.poly(_rand(ch, rng, S, N), S), E.poly(_rand(ch, rng, S, N), S)
    cs = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(4)]
    EA = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    EB = [E.poly(_rand(ch, rng, Sp, N), Sp) for _ in range(nd)]
    a0, a1 = E.poly(), E.poly()
    Xs = E.seeded(1, Sp, 5)[0]
    short = E.seeded(nd, sorted(ch.ctxt[:-1] + ch.special), 6)    # lacks the top ctxt prime
    Sarr = np.ascontiguousarray(np.array(S, dtype=np.int32))
    Sbad = np.ascontiguousarray(np.array(S + ch.special[:1], dtype=np.int32))

    def call(D=dg, maxdig=nd, nitems=1, S_=Sarr, C0=c0, C1=c1, p=17, k0=(1, 3), ea0=EA, k1=(1, 17), ea1=EA, eb1=EB,
             consts=None, consts1=False, kf=5, eaf=EA, ndig=nd, acc0=a0, acc1=a1, n0=None, n1=None):
        consts = consts if consts is not None else cs
        c1s = (cs if consts1 is False else consts1) if consts1 is not None else None
        return L.hb_block_linear_map(_pa(D), maxdig, nitems, S_.ctypes.data_as(C.POINTER(C.c_int32)), len(S_), _pa([C0]), _pa([C1]),
                                     C.c_uint64(p), len(k0) if n0 is None else n0, _u64(k0), _pa(list(ea0) * len(k0)),
                                     _pa(list(EB) * len(k0)), len(k1) if n1 is None else n1, _u64(k1), _pa(list(ea1) * len(k1)),
                                     _pa(list(eb1) * len(k1)), _pa(consts), _pa(c1s) if c1s is not None else None,
                                     C.c_uint64(kf), _pa(eaf), _pa(EB), ndig, _pa([acc0]), _pa([acc1]), 0)

    cases = [
        ("k0 = 2", HB_ERR_INDEX_SET, lambda: call(k0=(1, 2))),
        ("k1 = 0", HB_ERR_INDEX_SET, lambda: call(k1=(1, 0))),
        ("k1 = m", HB_ERR_INDEX_SET, lambda: call(k1=(1, 64))),
        ("kfinal = 4", HB_ERR_INDEX_SET, lambda: call(kf=4)),
        ("S with a special prime", HB_ERR_INDEX_SET, lambda: call(S_=Sbad)),
        ("seeded evk0_a without a needed row", HB_ERR_INDEX_SET, lambda: call(ea0=short)),
        ("seeded evkf_a without a needed row", HB_ERR_INDEX_SET, lambda: call(eaf=short)),
        ("n0 = 0", HB_ERR_BAD_ARG, lambda: call(n0=0)),
        ("n1 = 0", HB_ERR_BAD_ARG, lambda: call(n1=0)),
        ("nitems = 0", HB_ERR_BAD_ARG, lambda: call(nitems=0)),
        ("ptxt_space = 0", HB_ERR_BAD_ARG, lambda: call(p=0)),
        ("too few digit slots", HB_ERR_BAD_ARG, lambda: call(maxdig=nd - 1)),
        ("too few matrix columns", HB_ERR_BAD_ARG, lambda: call(ndig=nd - 1)),
        ("acc0 = c0", HB_ERR_BAD_ARG, lambda: call(acc0=c0)),
        ("acc1 = a digit", HB_ERR_BAD_ARG, lambda: call(acc1=dg[0])),
        ("acc0 = a block", HB_ERR_BAD_ARG, lambda: call(acc0=cs[2])),
        ("acc1 = a matrix row", HB_ERR_BAD_ARG, lambda: call(acc1=EB[0])),
        ("acc0 = acc1", HB_ERR_BAD_ARG, lambda: call(acc1=a0)),
        ("seeded c1", HB_ERR_BAD_ARG, lambda: call(C1=Xs)),
        ("seeded digit", HB_ERR_BAD_ARG, lambda: call(D=[Xs] + dg[1:])),
        ("seeded block", HB_ERR_BAD_ARG, lambda: call(consts=[Xs] + cs[1:])),
        ("seeded set-1 block", HB_ERR_BAD_ARG, lambda: call(consts1=cs[:3] + [Xs])),
        ("seeded evk1_b", HB_ERR_BAD_ARG, lambda: call(eb1=[Xs] + EB[1:])),
        ("seeded acc0", HB_ERR_BAD_ARG, lambda: call(acc0=Xs)),
    ]
    assert call() == 0, L.hb_last_error()
    for name, code, f in cases:
        E.sync()
        before = E.stats()["launches"]
        rc = f()
        assert rc == code, (name, rc, L.hb_last_error())
        assert E.stats()["launches"] == before, name
    # NULL blocks are zero blocks, and a native call needs no final amount
    assert call(consts=[None, cs[1], None, None], consts1=None, kf=4) == 0, L.hb_last_error()
    E.close()


# ---- 4. code generation

def test_hoist_kernel_keeps_its_state_in_registers(engine_codegen):
    ptx, report = engine_codegen
    frames = {k: v for k, v in _frames(report).items() if "k_ks_hoist" in k}
    assert len(frames) == 3, frames
    assert all(v == (0, 0, 0) for v in frames.values()), frames
    assert not {k: v for k, v in _depots(ptx).items() if "k_ks_hoist" in k}


# ---- 5. full size on the GPU: parity with the existing entry points and the step-by-step path, CUDA graph

def _full(cuda_lib, m, p, bits, c):
    from helib_b200 import Chain
    ch = Chain(m, p, 1, bits, c, lib=cuda_lib)
    E = Engine(ch.m, ch.primes, None, ch.digits, ch.special, lib=cuda_lib)
    return ch, E


def _full_case(E, ch, k0, k1, kf, bad, B, seed):
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    nd, n0, n1 = len(ch.digits), len(k0), len(k1)
    C0, C1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
    E.randomize(C0 + C1, S, seed)
    DG = E.break_into_digits(C1, S)
    CS = [[E.poly() for _ in range(n1)] for _ in range(n0)]
    CS1 = [[E.poly() for _ in range(n1)] for _ in range(n0)] if bad else None
    E.randomize([x for r in CS + (CS1 or []) for x in r], Sp, seed + 1)
    CS[n0 - 1][n1 - 1] = None

    def mats(ks, s):
        EA, EB, SA = [], [], []
        for j, k in enumerate(ks):
            if k == 1:
                EA.append(None); EB.append(None); SA.append(None)
                continue
            EA.append([E.poly() for _ in range(nd)]); EB.append([E.poly() for _ in range(nd)])
            E.randomize(EA[-1], Sp, s + j); E.randomize(EB[-1], Sp, s + 500 + j)
            SA.append(E.seeded(nd, Sp, s + j))
        return EA, EB, SA
    keys = [mats(k0, seed + 1000), mats(k1, seed + 2000), mats([kf], seed + 3000) if bad else ([None], [None], [None])]
    one = E.poly(np.ones((E.np, E.N), dtype=np.uint64), Sp)
    return DG, C0, C1, CS, CS1, keys, one


@pytest.mark.gpu
@pytest.mark.parametrize("dim", ["cfg5-dim0", "cfg5-dim1", "cfg5-dim2", "cfg3"])
def test_full_size_matches_the_engine_paths(cuda_lib, dim):
    """Config 5's ring (m = 21845, p = 2, d = 16) with its three dimensions' amounts, and config 3's (m = 2^17, p = 257)
    with 16 x 16 synthetic amounts, 3 ciphertexts: the fused call, with expanded and with seeded matrices, equals the
    existing entry points and the step-by-step engine path bit for bit."""
    if dim == "cfg3":
        ch, E = _full(cuda_lib, 1 << 17, 257, 1500, 3)
        gen, D, bad = 5, 16, False
    else:
        ch, E = _full(cuda_lib, 21845, 2, 580, 2)
        gen, D, bad = {"cfg5-dim0": (8996, 16, False), "cfg5-dim1": (17477, 4, False), "cfg5-dim2": (21591, 16, True)}[dim]
    p = ch.p
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    k0, k1, kf = amounts(ch.m, p, gen, D, 16)
    B = 3
    DG, C0, C1, CS, CS1, ((EA0, EB0, SA0), (EA1, EB1, SA1), (EAf, EBf, SAf)), one = _full_case(E, ch, k0, k1, kf, bad, B, 31)
    R0 = [[E.poly() for _ in k0] for _ in range(B)]
    R1 = [[E.poly() for _ in k0] for _ in range(B)]
    Y0, Y1, Z0, Z1 = ([E.poly() for _ in range(B)] for _ in range(4))
    tmp = [[E.poly() for _ in range(B)] for _ in range(5)]
    extra = dict(cs1=CS1, kf=kf, EAf=EAf[0], EBf=EBf[0]) if bad else {}
    refs = []
    for route in (existing_abi, step_by_step):
        A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        kw = dict(tmp=tmp, Z0=Z0, Z1=Z1) if route is step_by_step else {}
        route(E, DG, S, C0, C1, k0, EA0, EB0, k1, EA1, EB1, CS, A0, A1, p, R0=R0, R1=R1, Y0=Y0, Y1=Y1, one=one, **extra, **kw)
        refs.append([x.download(Sp)[Sp] for x in A0 + A1])
    assert all(np.array_equal(a, b) for a, b in zip(refs[0], refs[1]))
    for ka0, ka1, kaf in ((EA0, EA1, EAf), (SA0, SA1, SAf)):
        A0, A1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        E.block_linear_map(DG, S, C0, C1, k0, ka0, EB0, k1, ka1, EB1, CS, A0, A1, consts1=CS1, kfinal=kf, evkf_a=kaf[0],
                           evkf_b=EBf[0], ptxt_space=p)
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(refs[0], A0 + A1))
    E.close()


@pytest.mark.gpu
def test_config5_seeded_call_in_a_cuda_graph(cuda_lib):
    import torch
    ch, E = _full(cuda_lib, 21845, 2, 580, 2)
    S, Sp = ch.ctxt, sorted(ch.ctxt + ch.special)
    k0, k1, kf = amounts(ch.m, 2, 21591, 16, 16)
    DG, C0, C1, CS, CS1, ((_, EB0, SA0), (_, EB1, SA1), (_, EBf, SAf)), _ = _full_case(E, ch, k0, k1, kf, True, 2, 41)
    A0, A1 = [E.poly() for _ in range(2)], [E.poly() for _ in range(2)]

    def run():
        E.block_linear_map(DG, S, C0, C1, k0, SA0, EB0, k1, SA1, EB1, CS, A0, A1, consts1=CS1, kfinal=kf, evkf_a=SAf[0],
                           evkf_b=EBf[0], ptxt_space=2)
    run()
    ref = [x.download(Sp)[Sp] for x in A0 + A1]
    side = torch.cuda.Stream()
    torch.cuda.set_stream(side)
    E.set_stream(side.cuda_stream)
    run()   # warm on the capturing stream
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        run()
    for _ in range(2):
        for x in A0 + A1:
            x.upload(np.zeros((E.np, E.N), dtype=np.uint64), Sp)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert all(np.array_equal(a, x.download(Sp)[Sp]) for a, x in zip(ref, A0 + A1))
    torch.cuda.set_stream(torch.cuda.default_stream())
    E.close()


# ---- 6. the C++ mirror (tests/cpp/test_block_matmul.cpp): hb::BlockMatMul1D against the transcribed loop

def test_mirror_block_matmul_on_simulator():
    r = subprocess.run([build_exe("test_block_matmul", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "block matmul OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_block_matmul_on_gpu():
    r = subprocess.run([build_exe("test_block_matmul")], capture_output=True, text=True)
    assert r.returncode == 0 and "block matmul OK" in r.stdout, r.stdout + r.stderr
